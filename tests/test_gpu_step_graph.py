"""GPU: the learner step's stream schedule, read from its captured CUDA graph.

The step runs its weight re-pack, weight gradients and their reduces on lanes beside the caller's stream (kernels.h StepStreams).
A missing fork or join shows in the results only now and then, and an extra one only as a slower step, so these tests read the
schedule itself: each variant of the step is captured into a CUDA graph, and the graph's nodes and edges are read through the
driver API (cuGraphGetEdges_v2 reports each edge's type, so programmatic-launch edges are told apart from full ones).  The tests
require the data dependencies the kernels have, and the concurrency the schedule relies on.

`python -m tests.test_gpu_step_graph OUTDIR`, run from the repository root, writes the canonical text of every captured variant to
OUTDIR/<variant>.txt: the whole dependency DAG, for comparing two builds' schedules."""
import ctypes as C
import os
import re
import sys

import pytest
import torch

from oracle import impala_oracle as O

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------- graph reading
class _EdgeData(C.Structure):          # CUgraphEdgeData
    _fields_ = [('from_port', C.c_ubyte), ('to_port', C.c_ubyte), ('type', C.c_ubyte), ('reserved', C.c_ubyte * 5)]


class _KernelParams(C.Structure):      # CUDA_KERNEL_NODE_PARAMS_v2
    _fields_ = [('func', C.c_void_p), ('grid', C.c_uint * 3), ('block', C.c_uint * 3), ('shared', C.c_uint),
                ('params', C.c_void_p), ('extra', C.c_void_p), ('kern', C.c_void_p), ('ctx', C.c_void_p)]


class _MemsetParams(C.Structure):      # CUDA_MEMSET_NODE_PARAMS
    _fields_ = [('dst', C.c_uint64), ('pitch', C.c_size_t), ('value', C.c_uint), ('elem', C.c_uint), ('width', C.c_size_t),
                ('height', C.c_size_t)]


NODE_KERNEL, NODE_MEMCPY, NODE_MEMSET = 0, 1, 2


def _cu():
    cu = C.CDLL('libcuda.so.1')
    for f in ('cuGraphGetNodes', 'cuGraphGetEdges_v2', 'cuGraphNodeGetType', 'cuGraphKernelNodeGetParams_v2', 'cuGraphMemsetNodeGetParams',
              'cuFuncGetName', 'cuKernelGetName'):
        getattr(cu, f).restype = C.c_int
    return cu


def _ok(r, what):
    assert r == 0, f'{what}: CUresult {r}'


class StepGraph:
    """nodes (label, kind, memset destination), predecessors (node, edge type) and ancestor sets of a captured graph"""

    def __init__(self, g):
        cu = _cu()
        h = C.c_void_p(g.raw_cuda_graph())
        n = C.c_size_t(0)
        _ok(cu.cuGraphGetNodes(h, None, C.byref(n)), 'cuGraphGetNodes')
        nodes = (C.c_void_p * n.value)()
        _ok(cu.cuGraphGetNodes(h, nodes, C.byref(n)), 'cuGraphGetNodes')
        m = C.c_size_t(0)
        _ok(cu.cuGraphGetEdges_v2(h, None, None, None, C.byref(m)), 'cuGraphGetEdges_v2')
        fr, to, ed = (C.c_void_p * m.value)(), (C.c_void_p * m.value)(), (_EdgeData * m.value)()
        _ok(cu.cuGraphGetEdges_v2(h, fr, to, ed, C.byref(m)), 'cuGraphGetEdges_v2')
        index = {nodes[i]: i for i in range(n.value)}
        self.labels, self.kinds, self.dst = [], [], []
        for node in nodes:
            t = C.c_int()
            _ok(cu.cuGraphNodeGetType(C.c_void_p(node), C.byref(t)), 'cuGraphNodeGetType')
            dst = None
            if t.value == NODE_KERNEL:
                p = _KernelParams()
                _ok(cu.cuGraphKernelNodeGetParams_v2(C.c_void_p(node), C.byref(p)), 'cuGraphKernelNodeGetParams')
                name = C.c_char_p()
                if p.func:
                    _ok(cu.cuFuncGetName(C.byref(name), C.c_void_p(p.func)), 'cuFuncGetName')
                else:
                    _ok(cu.cuKernelGetName(C.byref(name), C.c_void_p(p.kern)), 'cuKernelGetName')
                label = (f'{name.value.decode()}<<<{",".join(map(str, p.grid))}|{",".join(map(str, p.block))}|{p.shared}>>>')
            elif t.value == NODE_MEMSET:
                p = _MemsetParams()
                _ok(cu.cuGraphMemsetNodeGetParams(C.c_void_p(node), C.byref(p)), 'cuGraphMemsetNodeGetParams')
                label, dst = f'memset {p.elem * p.width * p.height} B', p.dst
            elif t.value == NODE_MEMCPY:
                label = 'memcpy'
            else:
                label = f'node type {t.value}'
            self.labels.append(label)
            self.kinds.append(t.value)
            self.dst.append(dst)
        self.preds = [[] for _ in range(n.value)]
        for i in range(m.value):
            e = ed[i]
            kind = '' if (e.type, e.from_port, e.to_port) == (0, 0, 0) else f':{e.type}{e.from_port}{e.to_port}'
            self.preds[index[to[i]]].append((index[fr[i]], kind))
        self.order = self._topological()
        self.anc = [0] * n.value          # bit set of every node's ancestors
        for v in self.order:
            for u, _ in self.preds[v]:
                self.anc[v] |= self.anc[u] | (1 << u)

    def _topological(self):
        """deterministic topological order: among the ready nodes the least (label, predecessors' positions and edge types)"""
        succ = [[] for _ in self.labels]
        indeg = [len(p) for p in self.preds]
        for v, ps in enumerate(self.preds):
            for u, _ in ps:
                succ[u].append(v)
        ready, order, self.pos = [v for v in range(len(self.labels)) if indeg[v] == 0], [], {}
        while ready:
            v = min(ready, key=lambda x: (self.labels[x], sorted((self.pos[u], k) for u, k in self.preds[x])))
            ready.remove(v)
            self.pos[v] = len(order)
            order.append(v)
            for w in succ[v]:
                indeg[w] -= 1
                if indeg[w] == 0:
                    ready.append(w)
        assert len(order) == len(self.labels), 'the graph has a cycle'
        return order

    def canonical(self):
        """the whole DAG as text: one line per node in topological order, with its predecessors' line numbers and edge types"""
        return ''.join(f'{i} {self.labels[v]} <- {" ".join(f"{self.pos[u]}{k}" for u, k in sorted(self.preds[v], key=lambda e: (self.pos[e[0]], e[1])))}\n'
                       for i, v in enumerate(self.order))

    def find(self, key):
        """the kernel nodes of KERNELS[key] (every identifier of the key in the kernel's name), or the memset nodes into address `key`"""
        if isinstance(key, int):
            return [v for v, d in enumerate(self.dst) if d == key]
        idents = KERNELS[key]
        return [v for v, lab in enumerate(self.labels) if self.kinds[v] == NODE_KERNEL and all(_has_ident(lab, s) for s in idents)]

    def precedes(self, u, v):
        return bool(self.anc[v] >> u & 1)


def _has_ident(name, ident):
    """`ident` as a whole identifier of a mangled (length-prefixed) or demangled kernel name"""
    return f'{len(ident)}{ident}' in name or re.search(rf'(?<![A-Za-z0-9_]){ident}(?![A-Za-z0-9_])', name) is not None


KERNELS = {
    'obs_s2d': ('obs_s2d_kernel',), 'conv1_fwd': ('res_fwd_kernel', 'RConv1Fwd'), 'conv2_fwd': ('res_fwd_kernel', 'RConv2Fwd'),
    'enc_fused': ('enc_fused_fwd_kernel',), 'conv3_fwd': ('res_fwd_kernel', 'RConv3Fwd'), 'fc_fwd': ('igemm_tma_kernel', 'TFcFwd'),
    'pack': ('pack_weights_kernel',), 'column': ('column_step_kernel',), 'tail': ('impala_tail_warp_kernel',),
    'head_dh': ('head_bwd_dh_kernel',), 'dcore_to_dh': ('dcore_to_dh_kernel',),
    'head_wgrad': ('head_wgrad_kernel',), 'head_wgrad_reduce': ('head_wgrad_reduce_kernel',), 'a3_transpose': ('a3_transpose_kernel',),
    'fc_wgrad_bf16': ('igemm_tma_kernel', 'TFcWgradN'), 'fc_wgrad_split': ('igemm_tma_kernel', 'TFcWgrad'),
    'fc_dgrad': ('igemm_tma_kernel', 'TFcDgrad'),
    'conv3_wgrad': ('res_wgrad_kernel', 'RConv3Wgrad'), 'conv3_dgrad': ('res_fwd_kernel', 'RConv3Dgrad'),
    'conv2_wgrad': ('res_wgrad_kernel', 'RConv2Wgrad'), 'conv2_dgrad': ('res_fwd_kernel', 'RConv2Dgrad'),
    'conv1_wgrad': ('res_wgrad_kernel', 'RConv1Wgrad'),
    'reduce3': ('conv_wgrad_reduce_kernel', 'WgradReduce3'), 'reduce2': ('conv_wgrad_reduce_kernel', 'WgradReduce2'),
    'reduce1': ('conv_wgrad_reduce_kernel', 'WgradReduce1'),
    'clip_optim': ('clip_optim_kernel',), 'igemm_tma': ('igemm_tma_kernel',), 'res_wgrad': ('res_wgrad_kernel',),
}


# ---------------------------------------------------------------------------------------------------------------- captures
def _learner(T, B, A, use_lstm=False, **kw):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    sd = O.init_params(A, seed=3)
    if use_lstm:
        sd = {**sd, **O.init_lstm_params(A, seed=3)}
    return B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, use_lstm=use_lstm, **kw), init_state_dict=sd,
                             process_group=False)


def _batch(T, B, A):
    return {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=3, done_p=0.1).items()}


def _capture(L, fn):
    """the graph of fn() captured on the learner's capture stream (after one eager call: kernel attributes are set outside capture)"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g, stream=L._capture_stream()):
        fn()
    sg = StepGraph(g)
    del g
    return sg


def _lstm_actor_step(L, B, A):
    H = 513 + A
    dev = 'cuda'
    obs = torch.randint(0, 256, (1, B, 4, 84, 84), dtype=torch.uint8, device=dev)
    reward, done = torch.zeros(1, B, device=dev), torch.zeros(1, B, dtype=torch.uint8, device=dev)
    action = torch.zeros(1, B, dtype=torch.int64, device=dev)
    h_in, c_in = torch.zeros(2, B, H, device=dev), torch.zeros(2, B, H, device=dev)
    lg, bs = torch.empty(1, B, A, device=dev), torch.empty(1, B, device=dev)
    h_out, c_out = torch.empty_like(h_in), torch.empty_like(c_in)
    from scalerl_b200 import _lib
    lib = _lib.lib()
    _lib.check(lib.srl_learner_pack_weights(L._h, torch.cuda.current_stream().cuda_stream), 'pack_weights')
    return lambda: _lib.check(lib.srl_learner_forward_lstm_step(
        L._h, obs.data_ptr(), reward.data_ptr(), done.data_ptr(), action.data_ptr(), h_in.data_ptr(), c_in.data_ptr(), lg.data_ptr(),
        bs.data_ptr(), h_out.data_ptr(), c_out.data_ptr(), torch.cuda.current_stream().cuda_stream), 'forward_lstm_step')


STEP = (20, 32, 6)
LSTM_STEP = (5, 8, 6)
VARIANTS = {      # name: (shape, learner options, set_option switches)
    'default': (STEP, {}, {}),
    'fp32_split': (STEP, {'precision': 'fp32_split'}, {}),
    'column_fusion0': (STEP, {}, {'column_fusion': 0}),
    'fused_fwd1': (STEP, {}, {'fused_fwd': 1}),
    'lstm': (LSTM_STEP, {'use_lstm': True}, {}),
}


def capture_variant(name):
    """(StepGraph, learner) of one captured call.  The learner is open: the caller closes it."""
    if name in VARIANTS:
        (T, B, A), kw, opts = VARIANTS[name]
    else:
        (T, B, A), kw, opts = (LSTM_STEP, {'use_lstm': True}, {}) if name == 'lstm_actor_step' else (STEP, {}, {})
    L = _learner(T, B, A, **kw)
    for k, v in opts.items():
        L.set_option(k, v)
    dev = _batch(T, B, A)

    def step():
        L.forward_backward(dev)
        L.apply_gradients()
    fn = {'begin': lambda: L.forward_backward_begin(dev),
          'finish': lambda: L.backward_finish(dev),
          'forward': lambda: L.forward(dev)}.get(name, step)
    if name == 'lstm_actor_step':
        fn = _lstm_actor_step(L, B, A)
    if name == 'finish':
        L.forward_backward_begin(dev)
    return _capture(L, fn), L


def _one(G, key):
    v = G.find(key)
    assert v, f'no {key} node in the graph'
    return v


def _check_order(G, before, after):
    for a in before:
        for b in after:
            for u in _one(G, a):
                for v in _one(G, b):
                    assert G.precedes(u, v), f'{a} ({G.labels[u]}) must precede {b} ({G.labels[v]})'


def _check_unordered(G, first, second):
    for a in first:
        for b in second:
            for u in _one(G, a):
                for v in _one(G, b):
                    assert not G.precedes(u, v), f'{a} ({G.labels[u]}) must not be ordered before {b} ({G.labels[v]})'


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize('variant', ['default', 'fp32_split', 'column_fusion0', 'fused_fwd1', 'lstm'])
def test_step_graph_dependencies(variant):
    """what each kernel reads is written before it, and the lanes run beside the chain they were forked from"""
    G, L = capture_variant(variant)
    try:
        lstm, split, fused_front = variant == 'lstm', variant == 'fp32_split', variant == 'fused_fwd1'
        zero = L.flat_grads.data_ptr()            # the memset of the small gradients (everything before fc.weight)
        assert G.find(zero), 'no memset of the gradient buffer'
        fc_wgrad = 'fc_wgrad_split' if split else 'fc_wgrad_bf16'
        front, pack_reader = ('enc_fused', 'conv3_fwd') if fused_front else ('obs_s2d', 'conv2_fwd')
        reduces = ['reduce3', 'reduce2', 'reduce1']
        head = [] if lstm else ['head_wgrad', 'head_wgrad_reduce']
        if lstm:
            dh, dlogits = 'dcore_to_dh', None
        elif variant == 'column_fusion0':
            dh, dlogits = 'head_dh', 'tail'
        else:
            dh, dlogits = 'column', 'column'
        if not fused_front:
            _check_order(G, ['obs_s2d'], ['conv1_fwd'])
        _check_order(G, [front], ['conv1_wgrad'])
        _check_order(G, ['pack'], [pack_reader, 'fc_dgrad'])
        _check_order(G, [zero], head[1:] + [fc_wgrad] + reduces)
        _check_order(G, [dh], ['fc_dgrad', fc_wgrad])
        if not lstm:
            _check_order(G, [dlogits], ['head_wgrad'] + ([dh] if dh != dlogits else []))
            _check_order(G, ['head_wgrad'], ['head_wgrad_reduce'])
        if split:
            _check_order(G, ['conv3_fwd'], [fc_wgrad])
        else:
            _check_order(G, ['conv3_fwd'], ['a3_transpose'])
            _check_order(G, ['a3_transpose'], [fc_wgrad])
        _check_order(G, ['fc_dgrad'], ['conv3_wgrad', 'conv3_dgrad'])
        _check_order(G, ['conv3_dgrad'], ['conv2_wgrad', 'conv2_dgrad'])
        _check_order(G, ['conv2_dgrad'], ['conv1_wgrad'])
        for w, r in (('conv3_wgrad', 'reduce3'), ('conv2_wgrad', 'reduce2'), ('conv1_wgrad', 'reduce1')):
            _check_order(G, [w], [r])
        # the optimizer comes after every node but the copy of its norm behind it
        clip = _one(G, 'clip_optim')
        assert len(clip) == 1
        for v in range(len(G.labels)):
            if v != clip[0] and not G.precedes(clip[0], v):
                assert G.precedes(v, clip[0]), f'{G.labels[v]} must precede the optimizer'
        # concurrency: the re-pack runs beside the frame conversion, the wgrads beside the dgrad chain and beside each other
        _check_unordered(G, ['pack'], [front] + ([] if fused_front else ['conv1_fwd']))
        side = head + ([] if split else ['a3_transpose']) + [fc_wgrad, 'conv3_wgrad', 'reduce3', 'conv2_wgrad', 'reduce2']
        _check_unordered(G, side, ['fc_dgrad', 'conv3_dgrad', 'conv2_dgrad', 'conv1_wgrad'])
        _check_unordered(G, ['conv3_wgrad'], ['conv2_wgrad'])
        _check_unordered(G, ['conv2_wgrad'], ['conv3_wgrad'])
    finally:
        L.close()


def test_step_halves():
    """forward_backward_begin ends with the fc gradients, backward_finish holds the conv layers: each capture completing shows that
    every lane forked in it was joined (an unjoined stream fails the capture)"""
    G, L = capture_variant('begin')
    try:
        _one(G, 'fc_wgrad_bf16'), _one(G, 'fc_dgrad')
        for k in ('conv3_dgrad', 'conv2_dgrad', 'res_wgrad', 'reduce3', 'reduce2', 'reduce1'):
            assert not G.find(k), f'{k} in the first half'
    finally:
        L.close()
    G, L = capture_variant('finish')
    try:
        for k in ('conv3_wgrad', 'conv3_dgrad', 'conv2_wgrad', 'conv2_dgrad', 'conv1_wgrad', 'reduce3', 'reduce2', 'reduce1'):
            _one(G, k)
        assert not G.find('igemm_tma'), 'an fc kernel in the second half'
        _check_unordered(G, ['conv3_wgrad', 'reduce3', 'conv2_wgrad', 'reduce2'], ['conv3_dgrad', 'conv2_dgrad', 'conv1_wgrad'])
    finally:
        L.close()


# the profile slots one eager default step records (per-kernel profiling collapses every lane onto the caller's stream)
PROFILED_SLOTS = {'obs_s2d', 'conv1_fwd', 'conv2_fwd', 'conv3_fwd', 'fc_fwd', 'vtrace_loss_tail', 'zero_grads', 'head_bwd', 'fc_wgrad',
                  'fc_dgrad', 'conv3_wgrad', 'conv3_dgrad', 'conv2_wgrad', 'conv2_dgrad', 'conv1_wgrad', 'conv_wgrad_finalize', 'optimizer',
                  'pack_weights'}


def test_collapsed_step_matches_graph_step():
    """a profiled step runs every lane on the caller's stream, without PDL: the same bits as the captured step with lanes"""
    from scalerl_b200 import _lib
    lib = _lib.lib()
    T, B, A = STEP
    dev = _batch(T, B, A)
    P, Q = _learner(T, B, A), _learner(T, B, A)
    try:
        _lib.check(lib.srl_learner_set_profiling(P._h, 1), 'set_profiling')
        P.learn(dev, sync_stats=False, use_graph=False)       # eager: also sets the kernel attributes before Q's capture
        torch.cuda.synchronize()
        n = lib.srl_profile_slot_count()
        ms = (C.c_float * n)()
        _lib.check(lib.srl_learner_profile_collect(P._h, ms), 'profile_collect')
        recorded = {lib.srl_profile_slot_name(i).decode() for i in range(n) if ms[i] >= 0}
        assert recorded == PROFILED_SLOTS
        _lib.check(lib.srl_learner_set_profiling(P._h, 0), 'set_profiling')
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=Q._capture_stream()):
            Q.forward_backward(dev)
            Q.apply_gradients()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(P._losses, Q._losses)
        assert torch.equal(P.flat_grads, Q.flat_grads)
        assert torch.equal(P.flat_params, Q.flat_params)
        del g
    finally:
        P.close()
        Q.close()


if __name__ == '__main__':
    out = sys.argv[1]
    os.makedirs(out, exist_ok=True)
    for name in list(VARIANTS) + ['begin', 'finish', 'forward', 'lstm_actor_step']:
        G, L = capture_variant(name)
        L.close()
        with open(os.path.join(out, f'{name}.txt'), 'w') as f:
            f.write(G.canonical())
        print(name, len(G.labels), 'nodes')
