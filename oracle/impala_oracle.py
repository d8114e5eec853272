"""CPU oracle for the IMPALA learner hot path.  TEST INFRASTRUCTURE ONLY.

This file is a CPU restatement (torch-CPU fp32 + numpy fp64) of the arithmetic of the
reference's learner step.  It is imported ONLY by ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` -- never by the product path under
``scalerl_b200/``.  The product path fails loudly when the CUDA library is missing.

Parity pin: the reference ships no tests or golden vectors ("parity unpinned" by the reference's
own suite, SURVEY.md §8c).  The oracle is therefore pinned against outputs of the reference's own
importable modules run in the build container: ``oracle/make_golden.py`` imports
``/root/reference/scalerl/algorithms/impala/{vtrace,loss_fn}.py`` and
``/root/reference/scalerl/algorithms/utils/atari_model.py`` and writes ``tests/golden/*.npz``;
``tests/test_oracle_golden.py`` checks this file against those fixtures.

What each function follows (paths relative to /root/reference):
  * ``atari_forward``           scalerl/algorithms/utils/atari_model.py:77-143 (non-LSTM branch)
  * ``action_log_probs``        scalerl/algorithms/impala/vtrace.py:31-40
  * ``vtrace_from_importance_weights``  scalerl/algorithms/impala/vtrace.py:78-172
  * ``vtrace_from_logits``      scalerl/algorithms/impala/vtrace.py:43-75
  * ``impala_losses``           scalerl/algorithms/impala/loss_fn.py:5-23 and
                                scalerl/algorithms/impala/impala_atari.py:320-330
  * ``head_grads``              closed form of autograd through the above (SURVEY §8 a11)
  * ``learn_step``              scalerl/algorithms/impala/impala_atari.py:288-346
  * ``rmsprop_step``            torch.optim.RMSprop as constructed at impala_atari.py:99-105
  * ``adam_step``               torch.optim.Adam semantics (north_star's fused Adam); the reference's
                                only Adam is scalerl/algorithms/a3c/share_optim.py:94-120
  * ``clip_grad_norm``          torch.nn.utils.clip_grad_norm_ as called at impala_atari.py:344-345

``emulate_bf16=True`` rounds GEMM operands to bfloat16 at exactly the points where the CUDA path
does (weights, saved activations, back-propagated gradients), keeping fp32 accumulation.  It is used
to separate "kernel bug" from "bf16 operand rounding" in the parity tests.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

PARAM_ORDER = (
    'conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias',
    'fc.weight', 'fc.bias', 'policy.weight', 'policy.bias', 'baseline.weight', 'baseline.bias',
)


def param_shapes(num_actions: int) -> Dict[str, Tuple[int, ...]]:
    """Parameter shapes of AtariNet (atari_model.py:30-59), state_dict order, no LSTM."""
    core = 512 + num_actions + 1
    return {
        'conv1.weight': (32, 4, 8, 8), 'conv1.bias': (32,),
        'conv2.weight': (64, 32, 4, 4), 'conv2.bias': (64,),
        'conv3.weight': (64, 64, 3, 3), 'conv3.bias': (64,),
        'fc.weight': (512, 3136), 'fc.bias': (512,),
        'policy.weight': (num_actions, core), 'policy.bias': (num_actions,),
        'baseline.weight': (1, core), 'baseline.bias': (1,),
    }


def init_params(num_actions: int, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic (numpy) init with the distribution of torch's default Conv2d/Linear init:
    U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias.  numpy so the values do not depend on
    the torch version's RNG stream."""
    rng = np.random.RandomState(seed)
    out = {}
    shapes = param_shapes(num_actions)
    for name in PARAM_ORDER:
        shp = shapes[name]
        if name.endswith('.weight'):
            fan_in = int(np.prod(shp[1:]))
            last_fan_in = fan_in
        else:
            fan_in = last_fan_in
        bound = 1.0 / math.sqrt(fan_in)
        out[name] = torch.from_numpy(rng.uniform(-bound, bound, size=shp).astype(np.float32))
    return out


def synthetic_batch(T: int, B: int, A: int, seed: int = 0, done_p: float = 0.02) -> Dict[str, torch.Tensor]:
    """Synthetic [T+1, B] trajectory batch with the key schema of create_buffers
    (impala_atari.py:122-151); distributions from SURVEY.md §8(d).  numpy RNG for stability."""
    rng = np.random.RandomState(1000 + seed)
    obs = rng.randint(0, 256, size=(T + 1, B, 4, 84, 84), dtype=np.uint8)
    batch = {
        'obs': torch.from_numpy(obs),
        'reward': torch.from_numpy(rng.randn(T + 1, B).astype(np.float32)),
        'done': torch.from_numpy(rng.rand(T + 1, B) < done_p),
        'last_action': torch.zeros(T + 1, B, dtype=torch.int64),
        'action': torch.from_numpy(rng.randint(0, A, size=(T + 1, B)).astype(np.int64)),
        'episode_return': torch.from_numpy(rng.randn(T + 1, B).astype(np.float32)),
        'episode_step': torch.from_numpy(rng.randint(0, 1000, size=(T + 1, B)).astype(np.int32)),
        'policy_logits': torch.from_numpy(rng.randn(T + 1, B, A).astype(np.float32)),
        'baseline': torch.from_numpy(rng.randn(T + 1, B).astype(np.float32)),
    }
    return batch


def _bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(torch.float32)


# --------------------------------------------------------------------------------------------
# forward (atari_model.py:77-143, use_lstm=False)
# --------------------------------------------------------------------------------------------
def atari_forward(params: Dict[str, torch.Tensor], obs: torch.Tensor, reward: torch.Tensor,
                  action: torch.Tensor, emulate_bf16: bool = False, keep: bool = False):
    """obs u8 [T1,B,4,84,84], reward f32 [T1,B], action i64 [T1,B] -> (logits [T1,B,A], baseline [T1,B]).

    With emulate_bf16 the conv/fc operands are bf16-rounded like the CUDA path: the u8 frame is
    exact in bf16, conv1 multiplies raw u8 by bf16(W1) and applies 1/255 to the fp32 accumulator
    (instead of normalising the input, atari_model.py:94), activations are stored as bf16.
    """
    T1, B = obs.shape[:2]
    N = T1 * B
    rd = _bf16 if emulate_bf16 else (lambda t: t)
    x = obs.reshape(N, *obs.shape[2:]).to(params['conv1.weight'].dtype)      # float32, or float64 for fp64 references
    if emulate_bf16:
        a1 = F.conv2d(x, rd(params['conv1.weight']), None, stride=4) * (1.0 / 255.0) + params['conv1.bias'].view(1, -1, 1, 1)
    else:
        a1 = F.conv2d(x / 255.0, params['conv1.weight'], params['conv1.bias'], stride=4)
    a1 = rd(F.relu(a1))
    a2 = rd(F.relu(F.conv2d(a1, rd(params['conv2.weight']), params['conv2.bias'], stride=2)))
    a3 = rd(F.relu(F.conv2d(a2, rd(params['conv3.weight']), params['conv3.bias'], stride=1)))
    flat = a3.reshape(N, -1)
    h = F.relu(F.linear(flat, rd(params['fc.weight']), params['fc.bias']))  # fp32 (heads run fp32)
    A = params['policy.weight'].shape[0]
    one_hot = F.one_hot(action.reshape(N), A).float()
    clipped_reward = torch.clamp(reward, -1, 1).reshape(N, 1)
    core = torch.cat([h, clipped_reward, one_hot], dim=-1)
    logits = F.linear(core, params['policy.weight'], params['policy.bias'])
    baseline = F.linear(core, params['baseline.weight'], params['baseline.bias'])
    out = (logits.view(T1, B, A), baseline.view(T1, B))
    if keep:
        return out + (dict(x=x, a1=a1, a2=a2, a3=a3, h=h, core=core),)
    return out


# --------------------------------------------------------------------------------------------
# V-trace (vtrace.py)
# --------------------------------------------------------------------------------------------
def action_log_probs(policy_logits: torch.Tensor, actions: torch.Tensor) -> torch.Tensor:
    """vtrace.py:31-40: log_softmax(logits)[action]."""
    logp = F.log_softmax(policy_logits, dim=-1)
    return torch.gather(logp, -1, actions.unsqueeze(-1)).squeeze(-1)


def vtrace_from_importance_weights(log_rhos, discounts, rewards, values, bootstrap_value,
                                   clip_rho_threshold: Optional[float] = 1.0,
                                   clip_pg_rho_threshold: Optional[float] = 1.0):
    """vtrace.py:78-172, same dtype as the inputs (fp32 in the reference)."""
    rhos = torch.exp(log_rhos)
    clipped_rhos = torch.clamp(rhos, max=clip_rho_threshold) if clip_rho_threshold is not None else rhos
    cs = torch.clamp(rhos, max=1.0)
    values_tp1 = torch.cat([values[1:], bootstrap_value.unsqueeze(0)], dim=0)
    deltas = clipped_rhos * (rewards + discounts * values_tp1 - values)
    acc = torch.zeros_like(bootstrap_value)
    rows = []
    for t in range(discounts.shape[0] - 1, -1, -1):
        acc = deltas[t] + discounts[t] * cs[t] * acc
        rows.append(acc)
    rows.reverse()
    vs = torch.stack(rows) + values
    vs_tp1 = torch.cat([vs[1:], bootstrap_value.unsqueeze(0)], dim=0)
    pg_rhos = torch.clamp(rhos, max=clip_pg_rho_threshold) if clip_pg_rho_threshold is not None else rhos
    pg_adv = pg_rhos * (rewards + discounts * vs_tp1 - values)
    return vs, pg_adv


def vtrace_from_importance_weights_np64(log_rhos, discounts, rewards, values, bootstrap_value,
                                        clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0):
    """Independent float64 numpy witness of vtrace.py:135-169 (scalar recursion per column)."""
    log_rhos, discounts, rewards, values, bootstrap_value = [
        np.asarray(a, dtype=np.float64) for a in (log_rhos, discounts, rewards, values, bootstrap_value)]
    T, Bn = log_rhos.shape
    vs = np.zeros((T, Bn))
    pg = np.zeros((T, Bn))
    for b in range(Bn):
        acc = 0.0
        for t in range(T - 1, -1, -1):
            rho = math.exp(log_rhos[t, b])
            crho = min(rho, clip_rho_threshold) if clip_rho_threshold is not None else rho
            c = min(rho, 1.0)
            v_next = values[t + 1, b] if t + 1 < T else bootstrap_value[b]
            delta = crho * (rewards[t, b] + discounts[t, b] * v_next - values[t, b])
            acc = delta + discounts[t, b] * c * acc
            vs[t, b] = acc + values[t, b]
        for t in range(T):
            rho = math.exp(log_rhos[t, b])
            prho = min(rho, clip_pg_rho_threshold) if clip_pg_rho_threshold is not None else rho
            vs_next = vs[t + 1, b] if t + 1 < T else bootstrap_value[b]
            pg[t, b] = prho * (rewards[t, b] + discounts[t, b] * vs_next - values[t, b])
    return vs, pg


def vtrace_from_logits(behavior_policy_logits, target_policy_logits, actions, discounts, rewards,
                       values, bootstrap_value, clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0):
    """vtrace.py:43-75; returns (vs, pg_advantages, log_rhos, behavior_alp, target_alp)."""
    target_alp = action_log_probs(target_policy_logits, actions)
    behavior_alp = action_log_probs(behavior_policy_logits, actions)
    log_rhos = target_alp - behavior_alp
    vs, pg_adv = vtrace_from_importance_weights(log_rhos, discounts, rewards, values, bootstrap_value,
                                                clip_rho_threshold, clip_pg_rho_threshold)
    return vs, pg_adv, log_rhos, behavior_alp, target_alp


# --------------------------------------------------------------------------------------------
# losses (loss_fn.py) and their closed-form head gradients
# --------------------------------------------------------------------------------------------
def impala_losses(logits, actions, values, vs, pg_adv, baseline_cost, entropy_cost):
    """loss_fn.py:5-23 with the weights of impala_atari.py:320-330 -> (pg, baseline, entropy)."""
    logp = F.log_softmax(logits, dim=-1)
    p = F.softmax(logits, dim=-1)
    ce = -torch.gather(logp, -1, actions.unsqueeze(-1)).squeeze(-1)
    pg_loss = torch.sum(ce * pg_adv)
    baseline_loss = baseline_cost * 0.5 * torch.sum((vs - values) ** 2)
    entropy_loss = entropy_cost * torch.sum(p * logp)
    return pg_loss, baseline_loss, entropy_loss


def head_grads(logits, actions, values, vs, pg_adv, baseline_cost, entropy_cost):
    """d(total_loss)/d(logits), d(total_loss)/d(values) with vs, pg_adv detached:
       dlogits = adv*(p - onehot) + entropy_cost * p*(logp - sum(p*logp));  dV = -baseline_cost*(vs - V)."""
    logp = F.log_softmax(logits, dim=-1)
    p = logp.exp()
    onehot = F.one_hot(actions, logits.shape[-1]).to(logits.dtype)
    ent = torch.sum(p * logp, dim=-1, keepdim=True)
    dlogits = pg_adv.unsqueeze(-1) * (p - onehot) + entropy_cost * p * (logp - ent)
    dvalues = -baseline_cost * (vs - values)
    return dlogits, dvalues


# --------------------------------------------------------------------------------------------
# optimizer pieces
# --------------------------------------------------------------------------------------------
def clip_grad_norm(grads: Dict[str, torch.Tensor], max_norm: float) -> Tuple[float, float]:
    """clip_grad_norm_ (L2): coef = min(1, max_norm/(norm+1e-6)); scales grads in place."""
    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in grads.values():
        g.mul_(coef)
    return float(total), float(coef)


def rmsprop_step(params, grads, square_avg, lr, alpha, eps):
    """torch.optim.RMSprop, momentum=0, centered=False, weight_decay=0 (impala_atari.py:99-105):
       v = alpha*v + (1-alpha)*g^2 ; p -= lr * g / (sqrt(v) + eps)."""
    for k in params:
        g = grads[k]
        square_avg[k].mul_(alpha).addcmul_(g, g, value=1 - alpha)
        params[k].addcdiv_(g, square_avg[k].sqrt().add_(eps), value=-lr)


def adam_step(params, grads, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """torch.optim.Adam (no amsgrad/weight decay): bias-corrected; ``step`` is the 1-based count."""
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    for k in params:
        g = grads[k]
        exp_avg[k].mul_(beta1).add_(g, alpha=1 - beta1)
        exp_avg_sq[k].mul_(beta2).addcmul_(g, g, value=1 - beta2)
        denom = (exp_avg_sq[k].sqrt() / math.sqrt(bc2)).add_(eps)
        params[k].addcdiv_(exp_avg[k], denom, value=-lr / bc1)


# --------------------------------------------------------------------------------------------
# manual backward of the encoder (so operand rounding can be emulated)
# --------------------------------------------------------------------------------------------
def encoder_backward(params, saved, dlogits_full, dvalues_full, emulate_bf16=False):
    """Backward of atari_forward given d(loss)/d(logits) [N,A] and d(loss)/d(baseline) [N].
    Returns grads dict (fp32, PyTorch parameter layouts).  Mirrors autograd exactly in fp32 mode;
    in emulate_bf16 mode rounds the gradient/activation/weight operands of every tensor-core GEMM.
    """
    rd = _bf16 if emulate_bf16 else (lambda t: t)
    N = dlogits_full.shape[0]
    core, h, a3, a2, a1, x = saved['core'], saved['h'], saved['a3'], saved['a2'], saved['a1'], saved['x']
    g = {}
    # heads (fp32 CUDA cores in the product)
    g['policy.weight'] = dlogits_full.t() @ core
    g['policy.bias'] = dlogits_full.sum(0)
    g['baseline.weight'] = dvalues_full.view(1, N) @ core
    g['baseline.bias'] = dvalues_full.sum().view(1)
    dcore = dlogits_full @ params['policy.weight'] + dvalues_full.view(N, 1) * params['baseline.weight']
    dh = dcore[:, :512] * (h > 0).float()
    dh_op = rd(dh)
    # fc
    flat = a3.reshape(N, -1)
    g['fc.weight'] = dh_op.t() @ flat
    g['fc.bias'] = dh.sum(0) if not emulate_bf16 else dh_op.sum(0)
    da3 = (dh_op @ rd(params['fc.weight'])).view_as(a3) * (a3 > 0).float()
    da3_op = rd(da3)
    # conv3
    g['conv3.weight'] = torch.nn.grad.conv2d_weight(a2, params['conv3.weight'].shape, da3_op, stride=1)
    g['conv3.bias'] = da3_op.sum((0, 2, 3))
    da2 = torch.nn.grad.conv2d_input(a2.shape, rd(params['conv3.weight']), da3_op, stride=1) * (a2 > 0).float()
    da2_op = rd(da2)
    # conv2
    g['conv2.weight'] = torch.nn.grad.conv2d_weight(a1, params['conv2.weight'].shape, da2_op, stride=2)
    g['conv2.bias'] = da2_op.sum((0, 2, 3))
    da1 = torch.nn.grad.conv2d_input(a1.shape, rd(params['conv2.weight']), da2_op, stride=2) * (a1 > 0).float()
    da1_op = rd(da1)
    # conv1 (wgrad only); the 1/255 input normalisation is linear -> scale the result
    if emulate_bf16:
        g['conv1.weight'] = torch.nn.grad.conv2d_weight(x, params['conv1.weight'].shape, da1_op, stride=4) * (1.0 / 255.0)
    else:
        g['conv1.weight'] = torch.nn.grad.conv2d_weight(x / 255.0, params['conv1.weight'].shape, da1_op, stride=4)
    g['conv1.bias'] = da1_op.sum((0, 2, 3))
    return g


# --------------------------------------------------------------------------------------------
# the whole learner step (impala_atari.py:288-346)
# --------------------------------------------------------------------------------------------
DEFAULT_HP = dict(discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, reward_clipping='abs_one',
                  clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0, max_grad_norm=40.0,
                  learning_rate=1e-4, alpha=0.99, epsilon=1e-5, momentum=0.0,
                  optimizer='rmsprop', adam_beta1=0.9, adam_beta2=0.999, adam_eps=1e-8)


def learn_step(params: Dict[str, torch.Tensor], opt_state: Dict[str, Dict[str, torch.Tensor]],
               batch: Dict[str, torch.Tensor], hp: Optional[dict] = None, emulate_bf16: bool = False,
               use_autograd: bool = False, update: bool = True):
    """One learner step; mutates ``params`` / ``opt_state`` in place when ``update``.

    Returns a dict with logits, baseline, vs, pg_advantages, losses, grads (pre-clip), grad_norm,
    clip_coef and the stats of impala_atari.py:333-340.
    opt_state: {'square_avg': {...}} for rmsprop or {'exp_avg':..., 'exp_avg_sq':..., 'step': int}.
    """
    h = dict(DEFAULT_HP)
    if hp:
        h.update(hp)
    with torch.no_grad():
        T1, B = batch['obs'].shape[:2]
        T = T1 - 1
        A = params['policy.weight'].shape[0]
        if use_autograd:
            assert not emulate_bf16
            ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
            with torch.enable_grad():
                logits, baseline = atari_forward(ps, batch['obs'], batch['reward'], batch['action'])
        else:
            logits, baseline, saved = atari_forward(params, batch['obs'], batch['reward'], batch['action'],
                                                    emulate_bf16=emulate_bf16, keep=True)
        bootstrap_value = baseline[-1].detach()                                   # :293
        with torch.set_grad_enabled(use_autograd):
            tl, tv = logits[:-1], baseline[:-1]                                   # :297-300
        rewards = batch['reward'][1:]
        if h['reward_clipping'] == 'abs_one':                                     # :302-306
            rewards = torch.clamp(rewards, -1, 1)
        discounts = (~batch['done'][1:]).float() * h['discounting']               # :308
        actions = batch['action'][1:]
        vs, pg_adv, log_rhos, b_alp, t_alp = vtrace_from_logits(                  # :310-318
            batch['policy_logits'][1:], tl.detach(), actions, discounts, rewards, tv.detach(),
            bootstrap_value, h['clip_rho_threshold'], h['clip_pg_rho_threshold'])
        if use_autograd:
            with torch.enable_grad():
                pg_loss, baseline_loss, entropy_loss = impala_losses(
                    tl, actions, tv, vs, pg_adv, h['baseline_cost'], h['entropy_cost'])
                total = pg_loss + baseline_loss + entropy_loss
                total.backward()
            grads = {k: ps[k].grad.detach().clone() for k in PARAM_ORDER}
            logits, baseline = logits.detach(), baseline.detach()
            pg_loss, baseline_loss, entropy_loss = pg_loss.detach(), baseline_loss.detach(), entropy_loss.detach()
        else:
            pg_loss, baseline_loss, entropy_loss = impala_losses(
                tl, actions, tv, vs, pg_adv, h['baseline_cost'], h['entropy_cost'])
            dl, dv = head_grads(tl, actions, tv, vs, pg_adv, h['baseline_cost'], h['entropy_cost'])
            dl_full = torch.cat([dl, torch.zeros(1, B, A)], 0).reshape(T1 * B, A)  # row T dropped by [:-1]
            dv_full = torch.cat([dv, torch.zeros(1, B)], 0).reshape(T1 * B)
            grads = encoder_backward(params, saved, dl_full, dv_full, emulate_bf16=emulate_bf16)
        total_loss = pg_loss + baseline_loss + entropy_loss
        done = batch['done'][1:]
        ep_ret = batch['episode_return'][1:][done]                                # :332
        out = dict(policy_logits=logits, baseline=baseline, vs=vs, pg_advantages=pg_adv, log_rhos=log_rhos,
                   pg_loss=float(pg_loss), baseline_loss=float(baseline_loss), entropy_loss=float(entropy_loss),
                   total_loss=float(total_loss), episode_returns=tuple(ep_ret.numpy()),
                   mean_episode_return=float(torch.mean(ep_ret)) if ep_ret.numel() else float('nan'),
                   grads={k: v.clone() for k, v in grads.items()})
        gn, coef = clip_grad_norm(grads, h['max_grad_norm'])                      # :344-345
        out['grad_norm'], out['clip_coef'] = gn, coef
        if update:                                                                # :346
            if h['optimizer'] == 'rmsprop':
                rmsprop_step(params, grads, opt_state['square_avg'], h['learning_rate'], h['alpha'], h['epsilon'])
            else:
                opt_state['step'] += 1
                adam_step(params, grads, opt_state['exp_avg'], opt_state['exp_avg_sq'], opt_state['step'],
                          h['learning_rate'], h['adam_beta1'], h['adam_beta2'], h['adam_eps'])
        return out


# --------------------------------------------------------------------------------------------
# LSTM core (atari_model.py:52-55,61-75,109-120; use_lstm=True): 2-layer nn.LSTM(H, H), H = 513 + A,
# stepped one time step at a time with the state multiplied by (1 - done_t) BEFORE each step.
# --------------------------------------------------------------------------------------------
LSTM_PARAM_ORDER = tuple(f'rnn_layer.{w}_l{l}' for l in (0, 1) for w in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'))


def init_lstm_params(num_actions: int, seed: int = 0) -> Dict[str, torch.Tensor]:
    """numpy init with nn.LSTM's default distribution U(-1/sqrt(H), 1/sqrt(H)); names = nn.LSTM state_dict keys"""
    H = 513 + num_actions
    rng = np.random.RandomState(7000 + seed)
    k = 1.0 / math.sqrt(H)
    out = {}
    for name in LSTM_PARAM_ORDER:
        shp = (4 * H, H) if 'weight' in name else (4 * H,)
        out[name] = torch.from_numpy(rng.uniform(-k, k, size=shp).astype(np.float32))
    return out


def lstm_core_forward(lp: Dict[str, torch.Tensor], core: torch.Tensor, done: torch.Tensor, state):
    """core [T1,B,H], done bool [T1,B], state = (h [2,B,H], c [2,B,H]) -> (out [T1,B,H], new state).
    Gate order i,f,g,o (torch.nn.LSTM); atari_model.py:113-119 resets the state with notdone before every step."""
    T1, B, H = core.shape
    h = [state[0][0], state[0][1]]
    c = [state[1][0], state[1][1]]
    outs = []
    notdone = (~done).float()
    for t in range(T1):
        m = notdone[t].view(B, 1)
        x = core[t]
        for l in range(2):
            hp, cp = h[l] * m, c[l] * m
            g = F.linear(x, lp[f'rnn_layer.weight_ih_l{l}'], lp[f'rnn_layer.bias_ih_l{l}']) + \
                F.linear(hp, lp[f'rnn_layer.weight_hh_l{l}'], lp[f'rnn_layer.bias_hh_l{l}'])
            i, f, gg, o = g.chunk(4, dim=1)
            c[l] = torch.sigmoid(f) * cp + torch.sigmoid(i) * torch.tanh(gg)
            h[l] = torch.sigmoid(o) * torch.tanh(c[l])
            x = h[l]
        outs.append(x)
    return torch.stack(outs), (torch.stack(h), torch.stack(c))


def atari_forward_lstm(params, lp, obs, reward, action, done, state):
    """AtariNet.forward with use_lstm=True (fp32): conv encoder -> core -> 2-layer LSTM -> heads on the LSTM output"""
    T1, B = obs.shape[:2]
    N = T1 * B
    x = obs.reshape(N, *obs.shape[2:]).float() / 255.0
    a1 = F.relu(F.conv2d(x, params['conv1.weight'], params['conv1.bias'], stride=4))
    a2 = F.relu(F.conv2d(a1, params['conv2.weight'], params['conv2.bias'], stride=2))
    a3 = F.relu(F.conv2d(a2, params['conv3.weight'], params['conv3.bias'], stride=1))
    hfc = F.relu(F.linear(a3.reshape(N, -1), params['fc.weight'], params['fc.bias']))
    A = params['policy.weight'].shape[0]
    core = torch.cat([hfc, torch.clamp(reward, -1, 1).reshape(N, 1), F.one_hot(action.reshape(N), A).float()], dim=-1)
    out, new_state = lstm_core_forward(lp, core.view(T1, B, -1), done, state)
    flat = out.reshape(N, -1)
    logits = F.linear(flat, params['policy.weight'], params['policy.bias'])
    baseline = F.linear(flat, params['baseline.weight'], params['baseline.bias'])
    return logits.view(T1, B, A), baseline.view(T1, B), new_state


def learn_step_lstm(params, lp, batch, state, hp: Optional[dict] = None):
    """impala_atari.py:288-346 with use_lstm=True, fp32 autograd; returns losses, logits, vs and the gradients of BOTH
    parameter dicts (no optimizer update -- the update rule is layout-agnostic and tested separately)."""
    h = dict(DEFAULT_HP)
    if hp:
        h.update(hp)
    ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    ls = {k: v.detach().clone().requires_grad_(True) for k, v in lp.items()}
    logits, baseline, _ = atari_forward_lstm(ps, ls, batch['obs'], batch['reward'], batch['action'], batch['done'], state)
    bootstrap_value = baseline[-1].detach()
    tl, tv = logits[:-1], baseline[:-1]
    rewards = batch['reward'][1:]
    if h['reward_clipping'] == 'abs_one':
        rewards = torch.clamp(rewards, -1, 1)
    discounts = (~batch['done'][1:]).float() * h['discounting']
    actions = batch['action'][1:]
    with torch.no_grad():
        vs, pg_adv, *_ = vtrace_from_logits(batch['policy_logits'][1:], tl.detach(), actions, discounts, rewards, tv.detach(),
                                            bootstrap_value, h['clip_rho_threshold'], h['clip_pg_rho_threshold'])
    pg_loss, baseline_loss, entropy_loss = impala_losses(tl, actions, tv, vs, pg_adv, h['baseline_cost'], h['entropy_cost'])
    total = pg_loss + baseline_loss + entropy_loss
    total.backward()
    return dict(policy_logits=logits.detach(), baseline=baseline.detach(), vs=vs, pg_advantages=pg_adv,
                pg_loss=float(pg_loss), baseline_loss=float(baseline_loss), entropy_loss=float(entropy_loss), total_loss=float(total),
                grads={k: v.grad.detach().clone() for k, v in ps.items()}, lstm_grads={k: v.grad.detach().clone() for k, v in ls.items()})


def new_opt_state(params, optimizer='rmsprop'):
    z = lambda: {k: torch.zeros_like(v) for k, v in params.items()}
    if optimizer == 'rmsprop':
        return {'square_avg': z()}
    return {'exp_avg': z(), 'exp_avg_sq': z(), 'step': 0}
