"""fp64 references of the LSTM core's operations (csrc/lstm.cu), one step at a time, on whichever operands the caller passes.

Plain torch on either device: the GPU check (tests/test_gpu_lstm_exact.py) evaluates them on the bf16 operands the kernels read, in
float64 on the GPU; tests/test_lstm_ref_cpu.py proves them against autograd through oracle.impala_oracle.lstm_core_forward.

Layouts (the kernels', srl_lstm_core_debug_buffer): H = 513 + A is padded to Hp = 576 (a multiple of 64; the same Hp for every A in
[1, 31]); gate vectors are gate-major [4][Hp] (i, f, g, o), so a [4H] nn.LSTM vector's gate q, unit j sits at q*Hp + j; weights are
[4Hp][Hp] with the same row order.  Sequences are [T1][B][...]; m_t = 1 - done_t is [T1][B][1].  Padding is zero everywhere, and the
kernels write zero gate activations there (sigmoid(0) would be 0.5), which `activate(pre, H)` mirrors.

Comparisons reuse tests/layer_ref.py (rel_l2, nerr, compare_stored)."""
import torch

F64 = torch.float64
GATES = 4
BIAS_CHUNK = 64             # lstm_bias_part_kernel's rows per chunk (also the 64-row k-block of the weight-gradient GEMMs)

# element types of the rows srl_lstm_core_debug_buffer / srl_lstm_debug_buffer lend (every other row is float32)
ROW_DTYPE = {'xin0': torch.bfloat16, 'hm': torch.bfloat16, 'hbf': torch.bfloat16, 'Wih': torch.bfloat16, 'WihT': torch.bfloat16,
             'Whh': torch.bfloat16, 'WhhT': torch.bfloat16, 'dgates': torch.bfloat16, 'done': torch.uint8}
LAYER_ROWS = ('hm', 'hbf', 'Wih', 'WihT', 'Whh', 'WhhT', 'gates', 'cseq', 'hseq', 'dgates')
SHARED_ROWS = ('xin0', 'c_init', 'done', 'gx', 'r', 'dx', 'dwpad', 'dc', 'dhm', 'bias_part')


def row_dtype(name):
    return ROW_DTYPE.get(name, torch.float32)


# ------------------------------------------------------------------------------------------------ layouts
def hidden(A):
    return 513 + A


def padded(H):
    return (H + 63) // 64 * 64


def pad_cols(x, Hp):
    """[..., H] -> [..., Hp], zero padded"""
    return torch.nn.functional.pad(x, (0, Hp - x.shape[-1]))


def pad_gates(v, H, Hp):
    """nn.LSTM's [..., 4H] -> gate-major [..., 4Hp]"""
    return pad_cols(v.reshape(*v.shape[:-1], GATES, H), Hp).reshape(*v.shape[:-1], GATES * Hp)


def unpad_gates(v, H):
    """[..., 4Hp] -> [..., 4H]"""
    Hp = v.shape[-1] // GATES
    return v.reshape(*v.shape[:-1], GATES, Hp)[..., :H].reshape(*v.shape[:-1], GATES * H)


def gate_padding(v, H):
    """the padding columns [H, Hp) of every gate block of [..., 4Hp]"""
    Hp = v.shape[-1] // GATES
    return v.reshape(*v.shape[:-1], GATES, Hp)[..., H:]


def pad_weight(w, Hp):
    """nn.LSTM's [4H][H] -> [4Hp][Hp] (gate-major rows, zero padded)"""
    H = w.shape[1]
    return pad_cols(pad_gates(w.t(), H, Hp).t(), Hp)


def unpad_weight(w, H):
    """[4Hp][Hp] -> [4H][H]"""
    return unpad_gates(w[:, :H].t(), H).t()


# ------------------------------------------------------------------------------------------------ forward
def preact(xin, hm, Wih, Whh, bias):
    """gate pre-activations xin Wih^T + hm Whh^T + bias (bias = b_ih + b_hh in the same layout) for any leading dimensions"""
    return xin.to(F64) @ Wih.to(F64).t() + hm.to(F64) @ Whh.to(F64).t() + bias.to(F64)


def activate(pre, H=None):
    """(i, f, g, o) = (sigmoid, sigmoid, tanh, sigmoid) of the pre-activations; with H, the padding columns are zero as the kernel
    writes them"""
    i, f, g, o = pre.chunk(GATES, -1)
    a = torch.cat([torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)], -1)
    if H is not None:
        gate_padding(a, H).zero_()
    return a


def cell(gates, c_prev, m):
    """c_t = f (m_t c_{t-1}) + i g,  h_t = o tanh(c_t)"""
    i, f, g, o = gates.to(F64).chunk(GATES, -1)
    c = f * (m * c_prev.to(F64)) + i * g
    return c, o * torch.tanh(c)


def forward_layer(xin, Wih, Whh, bias, h0, c0, m, H=None):
    """one layer over T1 steps from its own results (no rounding): xin [T1][B][X] -> hm (the recurrent operand m_t h_{t-1}), gates, c, h"""
    hm, gates, cs, hs = [], [], [], []
    h, c = h0.to(F64), c0.to(F64)
    for t in range(xin.shape[0]):
        hm.append(m[t] * h)
        gates.append(activate(preact(xin[t], hm[t], Wih, Whh, bias), H))
        c, h = cell(gates[t], c, m[t])
        cs.append(c)
        hs.append(h)
    return tuple(torch.stack(v) for v in (hm, gates, cs, hs))


# ------------------------------------------------------------------------------------------------ backward
def bwd_step(gates, c, c_prev, m_t, dh, dc_in):
    """one BPTT cell step (lstm_cell_bwd_kernel): dh is this step's full dh (dh_out + m_{t+1} dhm_{t+1}), dc_in the carry from step
    t + 1 (dcT at the last step) -> (dgates [.., 4X], the carry into step t - 1 (masked by m_t))"""
    i, f, g, o = gates.to(F64).chunk(GATES, -1)
    tc = torch.tanh(c.to(F64))
    cp = m_t * c_prev.to(F64)
    dct = dh * o * (1 - tc * tc) + dc_in
    d = torch.cat([dct * g * i * (1 - i), dct * cp * f * (1 - f), dct * i * (1 - g * g), dh * tc * o * (1 - o)], -1)
    return d, m_t * dct * f


def bwd_step_terms(gates, c, c_prev, m_t, dh_terms, dc_terms):
    """bwd_step on |terms|: the sum of |terms| each output is made of, the scale of its fp32 rounding and cancellation"""
    i, f, g, o = gates.to(F64).abs().chunk(GATES, -1)
    tc = torch.tanh(c.to(F64)).abs()
    cp = m_t * c_prev.to(F64).abs()
    dct = dh_terms * o * (1 - tc * tc) + dc_terms
    d = torch.cat([dct * g * i * (1 - i), dct * cp * f * (1 - f), dct * i * (1 - g * g), dh_terms * tc * o * (1 - o)], -1)
    return d, m_t * dct * f


def recurrent_grad(dgates, Whh):
    """dhm_t = dgates_t Whh: the gradient w.r.t. the recurrent operand m_t h_{t-1}"""
    return dgates.to(F64) @ Whh.to(F64)


def input_grad(dgates, Wih):
    """dX = dgates Wih: the gradient w.r.t. the layer's input (dh_out of the layer below, or dcore)"""
    return dgates.to(F64) @ Wih.to(F64)


def bptt_layer(gates, cseq, c_init, m, dh_out, Whh, steps, dhT=None, dcT=None, dgates_next=None, dh_out_terms=None):
    """BPTT of one layer over steps [0, steps) in fp64.  dh_out [steps][B][X]; dhT / dcT [B][X] (None: zero) seed step steps-1: dhT
    is added to its dh unmasked and dcT is its incoming carry.  Every other step's dh adds m_{t+1} dhm_{t+1} with dhm_{t+1} =
    dgates_{t+1} Whh, taken from `dgates_next` where given (the GPU's stored dgates) and from this function's own otherwise.
    The dc carry is always this function's own.  -> dict(dgates [steps][B][4X], terms (sum |terms| of each, see bwd_step_terms),
    dh0 = m_0 dhm_0, dc0 = the carry out of step 0)"""
    B, X = c_init.shape
    z = torch.zeros(B, X, dtype=F64, device=c_init.device)
    dc = z if dcT is None else dcT.to(F64)
    dc_terms = dc.abs()
    dg, terms = [None] * steps, [None] * steps
    src = lambda t: dg[t] if dgates_next is None else dgates_next[t].to(F64)
    absW = Whh.to(F64).abs()
    for t in reversed(range(steps)):
        c_prev = c_init if t == 0 else cseq[t - 1]
        if t + 1 < steps:
            mn, nxt, nxt_terms = m[t + 1], recurrent_grad(src(t + 1), Whh), src(t + 1).abs() @ absW
        else:
            mn = 1.0
            nxt = z if dhT is None else dhT.to(F64)
            nxt_terms = nxt.abs()
        dh = dh_out[t].to(F64) + mn * nxt
        dh_terms = (dh_out[t].to(F64).abs() if dh_out_terms is None else dh_out_terms[t]) + mn * nxt_terms
        dg[t], dc = bwd_step(gates[t], cseq[t], c_prev, m[t], dh, dc)
        terms[t], dc_terms = bwd_step_terms(gates[t], cseq[t], c_prev, m[t], dh_terms, dc_terms)
    return {'dgates': torch.stack(dg), 'terms': torch.stack(terms), 'dh0': m[0] * recurrent_grad(src(0), Whh), 'dc0': dc}


def weight_grads(dgates, xin, hm, r0, r1):
    """dWih = dgates^T xin, dWhh = dgates^T hm and the bias gradient (column sums of dgates) over rows [r0, r1) of [NB][...] rows"""
    d = dgates[r0:r1].to(F64)
    return d.t() @ xin[r0:r1].to(F64), d.t() @ hm[r0:r1].to(F64), d.sum(0)


def mid_block(n, width=BIAS_CHUNK):
    """[lo, hi) of the middle width-wide block of n (the last block may be partial): one unit of work of a GEMM or the bias reduction"""
    nb = (n + width - 1) // width
    lo = nb // 2 * width
    return lo, min(n, lo + width)
