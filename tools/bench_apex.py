"""Learner steps/s and transitions/s of the Ape-X learner step (B200ApexLearner, captured, bf16 operands) against the reference's
statements (apex/worker.py:148-161) on torch/cuDNN with AtariQNet, eager and captured as a CUDA graph.  Each variant writes its
priorities into a GpuPrioritizedSampler of its own.  Rounds alternate between the variants; the median and range over rounds are
printed with the card's name and power limit, one JSON line per configuration.

With --dueling the learner runs the dueling head (ApexHParams(dueling_dqn=True)) beside the plain one, alternated in the same rounds,
and the torch statements use AtariQNet(A, dueling=True).  With --categorical it runs the categorical head (ApexHParams(categorical_dqn=True,
num_atoms=--atoms, v_min=-10, v_max=10)) beside the plain one, the torch statements become C51's (projection, cross-entropy, KL
priorities) on AtariQNet(A, categorical=True), and a last line gives the head kernels' times from torch.profiler at B = 512, A = 18
with their FLOP rate against the fp32 data-sheet rate (67 TFLOP/s).  With --quantile it runs the quantile learners
(ApexHParams(quantile_dqn=True, num_quantiles=N) for each N of --quantiles) and the categorical one at K = --atoms beside the plain one
(the torch statements stay the plain network's), and a last line per N gives the quantile head's kernel times at B = 512, A = 18.
With --noisy it runs the noisy learner (ApexHParams(noisy_dqn=True)) beside the plain one, the torch statements run on AtariQNet(A, noisy=True) with reset_noise() on the online and target network every
step, and a last line gives the noise kernels' times from torch.profiler at B = 512, A = 18 with the bytes they move against the HBM3
data-sheet bandwidth (3.35 TB/s).
With --dist-dueling it runs the categorical learner at K = --atoms and the quantile learners at each N of --quantiles, each beside
itself with the distributional dueling rows (ApexHParams(distributional_dueling=True)), alternated in the same rounds (the torch
statements stay the plain network's), and a last line per head gives the compose and decompose kernels' times from torch.profiler
with the bytes they move against the HBM3 data-sheet bandwidth, at B = 512, A = 18 and at the largest head, A = 31, K = 64.

    python tools/bench_apex.py [--rounds 5] [--steps 50] [--configs 32x6,32x18,512x6,512x18] [--dueling | --categorical [--atoms 51] | --noisy |
        --quantile [--quantiles 51,200] | --dist-dueling [--atoms 51] [--quantiles 51,200]]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scalerl_b200.algorithms.apex import ApexHParams, AtariQNet, B200ApexLearner, default_q_state_dict  # noqa: E402
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler  # noqa: E402

MEMORY = 4096        # sampler capacity: the sampled indices' range
V_MIN, V_MAX = -10.0, 10.0      # the categorical support (Atari rewards clipped to [-1, 1])


def card():
    """'<name>, <power limit>' as nvidia-smi reports them (the name alone when nvidia-smi is unavailable)"""
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def batch(B, A):
    g = torch.Generator(device='cuda').manual_seed(0)
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g)
    nobs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g)
    act = torch.randint(0, A, (B,), device='cuda', generator=g)
    rew = torch.randn(B, device='cuda', generator=g)
    done = torch.rand(B, device='cuda', generator=g) < 0.05
    w = torch.rand(B, device='cuda', generator=g)
    idxs = torch.randint(0, MEMORY, (B,), device='cuda', generator=g)
    return (obs, act, rew, nobs, done), w, idxs


def sampler():
    S = GpuPrioritizedSampler(MEMORY)
    S.add(MEMORY)
    return S


class TorchStep:
    """the reference's statements on torch/cuDNN (the priorities stay on the device and go into the GPU sampler).  The object owns
    every tensor the step reads or writes, so a captured replay of it stays valid as long as the object lives."""

    def __init__(self, B, A, exp, w, idxs, gamma=0.99, dueling=False, atoms=0, noisy=False):
        sd = default_q_state_dict(A, dueling=dueling, num_atoms=atoms, noisy=noisy)
        net = lambda: AtariQNet(A, dueling=dueling, categorical=atoms > 0, num_atoms=atoms or 51, v_min=V_MIN, v_max=V_MAX, noisy=noisy).cuda()
        self.noisy = noisy
        self.model, self.target, self.A, self.K = net(), net(), A, atoms
        self.rows = torch.arange(B, device='cuda')
        self.model.load_state_dict(sd)
        self.target.load_state_dict(sd)
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3, capturable=True)
        self.S, self.gamma, self.idxs = sampler(), gamma, idxs
        obs, act, rew, nobs, done = exp
        self.obs, self.nobs = obs, nobs
        self.actions, self.rewards, self.dones, self.weights = act.unsqueeze(1), rew.unsqueeze(1), done.float().unsqueeze(1), w.unsqueeze(1)
        self.prio = torch.empty(B, dtype=torch.float64, device='cuda')

    def __call__(self):
        if self.noisy:                  # new noise for both networks every update
            self.model.reset_noise()
            self.target.reset_noise()
        if self.K:
            return self.c51()
        current_q_values = self.model(self.obs).gather(1, self.actions)                       # worker.py:148
        with torch.no_grad():
            next_q_values = self.target(self.nobs).max(1, keepdim=True)[0]                    # :149
        target_q_values = self.rewards + (1 - self.dones) * self.gamma * next_q_values        # :150
        self.prio.copy_(torch.abs(current_q_values - target_q_values).detach().squeeze(1))    # :152-154
        loss = (self.weights * (current_q_values - target_q_values.detach()) ** 2).mean()     # :156-157
        self.opt.zero_grad(set_to_none=False)
        loss.backward()
        self.opt.step()
        self.S.update_priorities(self.idxs, self.prio, validate=False)

    def c51(self):
        """the categorical update (Bellemare et al. 2017, Algorithm 1) in torch statements, KL priorities"""
        A, K, z = self.A, self.K, self.model.support
        dz = z[1] - z[0]
        logp = F.log_softmax(self.model.q(self.model._features(self.obs)).view(-1, A, K), dim=2)[self.rows, self.actions[:, 0]]
        with torch.no_grad():
            pt = F.softmax(self.target.q(self.target._features(self.nobs)).view(-1, A, K), dim=2)
            pn = pt[self.rows, (pt * z).sum(2).argmax(1)]
            tz = (self.rewards + (1 - self.dones) * self.gamma * z).clamp(V_MIN, V_MAX)
            b = (tz - V_MIN) / dz
            lo, up = b.floor().long().clamp(0, K - 1), b.ceil().long().clamp(0, K - 1)
            m = torch.zeros_like(pn)
            m.scatter_add_(1, lo, pn * (up.float() - b) + pn * (lo == up).float())
            m.scatter_add_(1, up, pn * (b - lo.float()))
        ce = -(m * logp).sum(1)
        self.prio.copy_((torch.xlogy(m, m) - m * logp.detach()).sum(1).clamp(min=0))
        loss = (self.weights[:, 0] * ce).mean()
        self.opt.zero_grad(set_to_none=False)
        loss.backward()
        self.opt.step()
        self.S.update_priorities(self.idxs, self.prio, validate=False)


def head_profile(atoms, B=512, A=18, steps=20):
    """the categorical head's kernels in one captured learner step (torch.profiler over `steps` replays): mean µs per step and the
    GEMMs' FLOP rate against the fp32 data-sheet rate"""
    from torch.profiler import ProfilerActivity, profile
    exp, w, idxs = batch(B, A)
    L, S = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, categorical_dqn=True, num_atoms=atoms, v_min=V_MIN, v_max=V_MAX)), sampler()
    step = lambda: L.learn(exp, weights=w, idxs=idxs, sampler=S, sync_stats=False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    R = A * atoms
    flops = {'cat_gemm_kernel<false>': 2.0 * B * R * 512 * 2, 'cat_gemm_kernel<true>': 2.0 * B * R * 513}    # two logit sets: s, s' target
    out, total = {}, 0.0
    for e in prof.key_averages():
        if 'cat_' not in e.key:
            continue
        us = e.device_time_total / steps
        name = 'cat_gemm_kernel<true>' if 'Lb1' in e.key or '<true>' in e.key else ('cat_gemm_kernel<false>' if 'gemm' in e.key else e.key.split('(')[0])
        out[name] = {'us_per_step': us}
        if name in flops:
            out[name]['tflops'] = flops[name] / us * 1e-6
            out[name]['fraction_of_67_tflops'] = flops[name] / us * 1e-6 / 67.0
        total += us
    step_us = 1e6 / timed(step, 50)
    L.release_graphs()
    L.close()
    return {'card': card(), 'B': B, 'A': A, 'K': atoms, 'head_kernels': out, 'head_us_per_step': total, 'step_us': step_us,
            'head_share_of_step': total / step_us}


def quantile_profile(N, B=512, A=18, steps=20):
    """the quantile head's kernels in one captured learner step (torch.profiler over `steps` replays): mean µs per step, the GEMMs'
    FLOP rate against the fp32 data-sheet rate and the tail's quantile pairs per second"""
    from torch.profiler import ProfilerActivity, profile
    exp, w, idxs = batch(B, A)
    L, S = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, quantile_dqn=True, num_quantiles=N)), sampler()
    step = lambda: L.learn(exp, weights=w, idxs=idxs, sampler=S, sync_stats=False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    R = A * N
    flops = {'cat_gemm_kernel<false>': 2.0 * B * R * 512 * 2, 'cat_gemm_kernel<true>': 2.0 * B * R * 513}    # two quantile sets: s, s' target
    out, total = {}, 0.0
    for e in prof.key_averages():
        if 'cat_gemm' not in e.key and 'qr_tail' not in e.key:
            continue
        us = e.device_time_total / steps
        name = 'qr_tail_kernel' if 'qr_tail' in e.key else ('cat_gemm_kernel<true>' if 'Lb1' in e.key or '<true>' in e.key else 'cat_gemm_kernel<false>')
        out[name] = {'us_per_step': us}
        if name in flops:
            out[name]['tflops'] = flops[name] / us * 1e-6
            out[name]['fraction_of_67_tflops'] = flops[name] / us * 1e-6 / 67.0
        else:
            out[name]['quantile_pairs_per_s'] = B * N * N / us * 1e6
        total += us
    step_us = 1e6 / timed(step, 50)
    L.release_graphs()
    L.close()
    return {'card': card(), 'B': B, 'A': A, 'N': N, 'head_kernels': out, 'head_us_per_step': total, 'step_us': step_us,
            'head_share_of_step': total / step_us}


def noisy_profile(B=512, A=18, steps=20):
    """the noise kernels in one captured noisy learner step (torch.profiler over `steps` replays): mean µs per step, the bytes each
    moves (from the shapes) and its share of the HBM3 data-sheet bandwidth"""
    from torch.profiler import ProfilerActivity, profile
    exp, w, idxs = batch(B, A)
    L, S = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, noisy_dqn=True)), sampler()
    step = lambda: L.learn(exp, weights=w, idxs=idxs, sampler=S, sync_stats=False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    weights = 4 * (512 * 3136 + 512 + A * 512 + A)          # one fp32 copy of the noisy layers' weights and biases
    nn = 3136 + 512 + 512 + A
    nbytes = {'noisy_draw_kernel': 2 * 2 * nn * 4,        # two networks' normals and noise
              'noisy_compose_kernel': 2 * (3 * weights + 2 * nn * 4),    # per network: mu, sigma read, W written
              'noisy_sigma_grad_kernel': 2 * weights + nn * 4}          # dmu read, dsigma written
    out, total = {}, 0.0
    for e in prof.key_averages():
        name = next((k for k in nbytes if k in e.key), None)
        if name is None:
            continue
        us = e.device_time_total / steps
        out[name] = {'us_per_step': us, 'bytes': nbytes[name], 'tb_per_s': nbytes[name] / us * 1e-6,
                     'fraction_of_3_35_tb_per_s': nbytes[name] / us * 1e-6 / 3.35}
        total += us
    step_us = 1e6 / timed(step, 50)
    L.release_graphs()
    L.close()
    return {'card': card(), 'B': B, 'A': A, 'noise_kernels': out, 'noise_us_per_step': total, 'step_us': step_us,
            'noise_share_of_step': total / step_us}


def dist_dueling_profile(kind, W, B=512, A=18, steps=20):
    """the distributional dueling head's compose and decompose kernels in one captured learner step (torch.profiler over `steps`
    replays): mean µs per step, the bytes each moves (from the shapes) and its share of the HBM3 data-sheet bandwidth"""
    from torch.profiler import ProfilerActivity, profile
    exp, w, idxs = batch(B, A)
    head = dict(categorical_dqn=True, num_atoms=W, v_min=V_MIN, v_max=V_MAX) if kind == 'categorical' else dict(quantile_dqn=True, num_quantiles=W)
    L, S = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, distributional_dueling=True, **head)), sampler()
    step = lambda: L.learn(exp, weights=w, idxs=idxs, sampler=S, sync_stats=False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    params, rows = 4 * (W + A * W) * 513, 4 * A * W * 513       # value and advantage weights and biases; the composed rows
    nbytes = {'dist_dueling_compose_kernel': 2 * (params + rows),    # online and target: value and advantage read, rows written
              'dist_dueling_grad_kernel': rows + params}             # the rows' gradient read, the value and advantage gradients written
    out, total = {}, 0.0
    for e in prof.key_averages():
        name = next((k for k in nbytes if k in e.key), None)
        if name is None:
            continue
        us = e.device_time_total / steps
        out[name] = {'us_per_step': us, 'bytes': nbytes[name], 'tb_per_s': nbytes[name] / us * 1e-6,
                     'fraction_of_3_35_tb_per_s': nbytes[name] / us * 1e-6 / 3.35}
        total += us
    step_us = 1e6 / timed(step, 50)
    L.release_graphs()
    L.close()
    return {'card': card(), 'B': B, 'A': A, 'head': kind, 'W': W, 'dueling_row_kernels': out, 'dueling_rows_us_per_step': total,
            'step_us': step_us, 'dueling_rows_share_of_step': total / step_us}


class Captured:
    """a CUDA graph of `step` (warmed up on a side stream first); holds `step`, whose tensors the graph reads and writes"""

    def __init__(self, step):
        self.step = step
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                step()
        torch.cuda.current_stream().wait_stream(s)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            step()

    def __call__(self):
        self.graph.replay()


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--configs', default='32x6,32x18,512x6,512x18')
    ap.add_argument('--dueling', action='store_true', help='add the dueling learner and run the torch statements on the dueling net')
    ap.add_argument('--categorical', action='store_true', help='add the categorical learner and run C51 in torch statements')
    ap.add_argument('--atoms', type=int, default=51)
    ap.add_argument('--noisy', action='store_true', help='add the noisy learner and run the torch statements on the noisy net')
    ap.add_argument('--quantile', action='store_true', help='add the quantile learners and the categorical one at --atoms beside them')
    ap.add_argument('--quantiles', default='51,200', help='the quantile learners\' num_quantiles (--quantile, --dist-dueling)')
    ap.add_argument('--dist-dueling', action='store_true', help='the categorical and quantile learners with and without the distributional '
                    'dueling rows')
    a = ap.parse_args()
    if a.dueling + a.categorical + a.noisy + a.quantile + a.dist_dueling > 1:
        sys.exit('--dueling, --categorical, --noisy, --quantile and --dist-dueling are separate comparisons: pass one')
    atoms = a.atoms if a.categorical else 0
    quantiles = [int(x) for x in a.quantiles.split(',')] if a.quantile else []
    dd_heads = []           # --dist-dueling: (name, ApexHParams head keywords) of each head, run without and with the dueling rows
    if a.dist_dueling:
        dd_heads = [(f'categorical_K{a.atoms}', dict(categorical_dqn=True, num_atoms=a.atoms, v_min=V_MIN, v_max=V_MAX))] + \
            [(f'quantile_N{N}', dict(quantile_dqn=True, num_quantiles=int(N))) for N in a.quantiles.split(',')]
    if not torch.cuda.is_available():
        sys.exit('bench_apex.py measures on a CUDA device; none is present')
    name = card()
    for cfg in a.configs.split(','):
        B, A = (int(x) for x in cfg.split('x'))
        exp, w, idxs = batch(B, A)
        L, S = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A)), sampler()
        variants = {'b200_captured': lambda: L.learn(exp, weights=w, idxs=idxs, sampler=S, sync_stats=False)}
        learners = [L]
        if a.dueling:
            LD, SD = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, dueling_dqn=True)), sampler()
            learners.append(LD)
            variants['b200_dueling_captured'] = lambda: LD.learn(exp, weights=w, idxs=idxs, sampler=SD, sync_stats=False)
        if atoms:
            LC = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, categorical_dqn=True, num_atoms=atoms, v_min=V_MIN, v_max=V_MAX))
            SC = sampler()
            learners.append(LC)
            variants['b200_categorical_captured'] = lambda: LC.learn(exp, weights=w, idxs=idxs, sampler=SC, sync_stats=False)
        if a.noisy:
            LN, SN = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, noisy_dqn=True)), sampler()
            learners.append(LN)
            variants['b200_noisy_captured'] = lambda: LN.learn(exp, weights=w, idxs=idxs, sampler=SN, sync_stats=False)
        if quantiles:
            LC = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, categorical_dqn=True, num_atoms=a.atoms, v_min=V_MIN, v_max=V_MAX))
            learners.append(LC)
            variants[f'b200_categorical_K{a.atoms}_captured'] = (lambda L_, S_: lambda: L_.learn(exp, weights=w, idxs=idxs, sampler=S_,
                                                                                               sync_stats=False))(LC, sampler())
        for N in quantiles:
            LQ = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, quantile_dqn=True, num_quantiles=N))
            learners.append(LQ)
            variants[f'b200_quantile_N{N}_captured'] = (lambda L_, S_: lambda: L_.learn(exp, weights=w, idxs=idxs, sampler=S_,
                                                                                       sync_stats=False))(LQ, sampler())
        for hname, kw in dd_heads:
            for dd in (False, True):
                LH = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, distributional_dueling=dd, **kw))
                learners.append(LH)
                variants[f'b200_{hname}{"_dist_dueling" if dd else ""}_captured'] = \
                    (lambda L_, S_: lambda: L_.learn(exp, weights=w, idxs=idxs, sampler=S_, sync_stats=False))(LH, sampler())
        variants['torch_eager'] = TorchStep(B, A, exp, w, idxs, dueling=a.dueling, atoms=atoms, noisy=a.noisy)
        variants['torch_captured'] = Captured(TorchStep(B, A, exp, w, idxs, dueling=a.dueling, atoms=atoms, noisy=a.noisy))
        for fn in variants.values():           # warm-up: the learner's first call runs eagerly, the second captures
            for _ in range(3):
                fn()
        rates = {k: [] for k in variants}
        for _ in range(a.rounds):
            for k, fn in variants.items():
                rates[k].append(timed(fn, a.steps))
        torch_net = 'dueling' if a.dueling else (f'categorical K={atoms}' if atoms else ('noisy' if a.noisy else 'plain'))
        out = {'card': name, 'B': B, 'A': A, 'precision': 'bf16', 'torch_net': torch_net, 'rounds': a.rounds,
               'steps_per_round': a.steps}
        for k, r in rates.items():
            r = sorted(r)
            out[k] = {'steps_per_s_median': r[len(r) // 2], 'steps_per_s_range': [r[0], r[-1]],
                      'transitions_per_s_median': r[len(r) // 2] * B}
        print(json.dumps(out), flush=True)
        del variants
        for x in learners:
            x.release_graphs()
            x.close()
    if atoms:
        print(json.dumps(head_profile(atoms)), flush=True)
    if a.noisy:
        print(json.dumps(noisy_profile()), flush=True)
    for N in quantiles:
        print(json.dumps(quantile_profile(N)), flush=True)
    if a.dist_dueling:
        for kind, W in [('categorical', a.atoms)] + [('quantile', int(N)) for N in a.quantiles.split(',')]:
            print(json.dumps(dist_dueling_profile(kind, W)), flush=True)
        print(json.dumps(dist_dueling_profile('categorical', 64, A=31)), flush=True)


if __name__ == '__main__':
    main()
