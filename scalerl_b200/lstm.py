"""B200LstmCore -- the 2-layer LSTM core of AtariNet(use_lstm=True) (reference: scalerl/algorithms/utils/atari_model.py:
52-55,61-75,109-120) on the sm_90a kernels of csrc/lstm.cu.  Parameter names are nn.LSTM's state_dict keys
(``rnn_layer.weight_ih_l0`` ...), so checkpoints interchange with the reference model."""
import ctypes as C
from collections import OrderedDict
from typing import Dict, Tuple

import torch

from . import _lib

LSTM_PARAM_NAMES = tuple(f'rnn_layer.{w}_l{l}' for l in (0, 1) for w in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'))


class B200LstmCore:
    def __init__(self, T1: int, B: int, H: int, state_dict: Dict[str, torch.Tensor] = None, device=None, seed: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError('B200LstmCore needs a CUDA device (no CPU fallback)')
        self.T1, self.B, self.H = T1, B, H
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        g = torch.Generator().manual_seed(seed)
        k = 1.0 / H ** 0.5
        self.params, self.grads = OrderedDict(), OrderedDict()
        for n in LSTM_PARAM_NAMES:
            shp = (4 * H, H) if 'weight' in n else (4 * H,)
            v = state_dict[n].float() if state_dict is not None else (torch.rand(shp, generator=g) * 2 - 1) * k
            if tuple(v.shape) != shp:
                raise ValueError(f'{n}: shape {tuple(v.shape)} != {shp}')
            self.params[n] = v.to(self.device).contiguous()
            self.grads[n] = torch.zeros(shp, device=self.device)
        wp = (C.c_void_p * 8)(*[self.params[n].data_ptr() for n in LSTM_PARAM_NAMES])
        gp = (C.c_void_p * 8)(*[self.grads[n].data_ptr() for n in LSTM_PARAM_NAMES])
        h = C.c_void_p()
        self._L = _lib.lib()
        _lib.check(self._L.srl_lstm_create(T1, B, H, wp, gp, C.byref(h)), 'srl_lstm_create')
        self._h = h

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def zero_grad(self):
        for g in self.grads.values():
            g.zero_()

    @torch.no_grad()
    def forward(self, core: torch.Tensor, done: torch.Tensor, state: Tuple[torch.Tensor, torch.Tensor]):
        """core f32 [T1,B,H], done bool/u8 [T1,B], state (h, c) each f32 [2,B,H] -> (out [T1,B,H], (hT, cT))"""
        T1, B, H = self.T1, self.B, self.H
        if tuple(core.shape) != (T1, B, H) or core.dtype != torch.float32 or not core.is_cuda:
            raise ValueError(f'core must be a CUDA float32 tensor of shape {(T1, B, H)}')
        d = done.contiguous()
        d = d.view(torch.uint8) if d.dtype == torch.bool else d
        h0, c0 = [s.to(self.device, torch.float32).contiguous() for s in state]
        if tuple(h0.shape) != (2, B, H) or tuple(c0.shape) != (2, B, H):
            raise ValueError(f'state tensors must be {(2, B, H)}')
        out = torch.empty(T1, B, H, device=self.device)
        hT, cT = torch.empty(2, B, H, device=self.device), torch.empty(2, B, H, device=self.device)
        self._done = d
        _lib.check(self._L.srl_lstm_forward(self._h, core.contiguous().data_ptr(), d.data_ptr(), h0.data_ptr(), c0.data_ptr(), out.data_ptr(),
                                            hT.data_ptr(), cT.data_ptr(), self._stream()), 'srl_lstm_forward')
        return out, (hT, cT)

    @torch.no_grad()
    def backward(self, dout: torch.Tensor) -> torch.Tensor:
        """dout f32 [T1-1,B,H] -> dcore f32 [T1-1,B,H]; parameter gradients are accumulated into self.grads"""
        T, B, H = self.T1 - 1, self.B, self.H
        if tuple(dout.shape) != (T, B, H):
            raise ValueError(f'dout must be {(T, B, H)}')
        dcore = torch.empty(T, B, H, device=self.device)
        _lib.check(self._L.srl_lstm_backward(self._h, dout.contiguous().data_ptr(), self._done.data_ptr(), dcore.data_ptr(), self._stream()),
                   'srl_lstm_backward')
        return dcore

    def close(self):
        if getattr(self, '_h', None) is not None:
            self._L.srl_lstm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
