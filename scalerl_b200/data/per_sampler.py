"""GpuPrioritizedSampler -- device-side replacement of the segment-tree arithmetic of the reference's
PrioritizedReplayBuffer (scalerl/data/replay_buffer.py:276-381; trees: scalerl/data/segment_tree.py).  Same method
names/semantics for the priority bookkeeping (``add`` = ``_add``'s tree part, ``update_priorities``, ``sample`` ->
(idxs, weights)); transition storage is left to the caller (e.g. device tensors indexed by the returned ``idxs``)."""
import ctypes as C

import torch

from .. import _lib


class GpuPrioritizedSampler:
    def __init__(self, memory_size: int, alpha: float = 0.6, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError('GpuPrioritizedSampler needs a CUDA device (no CPU fallback)')
        self.memory_size, self.alpha = int(memory_size), float(alpha)
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._L = _lib.lib()
        h = C.c_void_p()
        _lib.check(self._L.srl_per_create(self.memory_size, self.alpha, C.byref(h)), 'srl_per_create')
        self._h = h
        self._invalid_seen = 0
        self._owned = True

    @classmethod
    def _view(cls, handle, memory_size: int, alpha: float, device):
        """the sampler over trees another object owns (GpuPrioritizedReplayBuffer's): close() leaves them to their owner"""
        s = cls.__new__(cls)
        s.memory_size, s.alpha, s.device = int(memory_size), float(alpha), torch.device(device)
        s._L, s._h, s._invalid_seen, s._owned = _lib.lib(), handle, 0, False
        return s

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def __len__(self):
        return int(self._L.srl_per_size(self._h))

    @property
    def capacity(self):
        return int(self._L.srl_per_capacity(self._h))

    def add(self, n: int = 1):
        """n new transitions enter with priority max_priority ** alpha (replay_buffer.py:318-322)"""
        _lib.check(self._L.srl_per_add(self._h, int(n), self._stream()), 'srl_per_add')

    def update_priorities(self, idxs: torch.Tensor, priorities: torch.Tensor, validate: bool = True):
        """replay_buffer.py:346-351.  The reference asserts ``priority > 0`` and ``0 <= idx < len(self)``; with ``validate``
        (default) a violation raises AssertionError-like ValueError after the launch (one 8-byte D2H read + stream sync);
        the kernel itself never writes out of bounds (invalid pairs are skipped) so ``validate=False`` is safe and sync-free."""
        idxs = idxs.to(self.device, torch.int64).contiguous()
        pr = priorities.to(self.device, torch.float64).contiguous()
        if idxs.numel() != pr.numel():
            raise ValueError('idxs and priorities must have the same length')
        _lib.check(self._L.srl_per_update_priorities(self._h, idxs.data_ptr(), pr.data_ptr(), idxs.numel(), self._stream()), 'srl_per_update_priorities')
        if validate:
            bad = int(self._L.srl_per_invalid_updates(self._h, self._stream()))
            if bad != self._invalid_seen:
                n_new, self._invalid_seen = bad - self._invalid_seen, bad
                raise ValueError(f'update_priorities: {n_new} pair(s) with idx outside [0, {len(self)}) or priority <= 0 were skipped')

    def sample(self, batch_size: int, beta: float = 0.4, uniforms: torch.Tensor = None, generator=None):
        """-> (idxs int64 [batch], weights float32 [batch]); ``uniforms`` (float64 in [0,1)) may be supplied for reproducibility"""
        if uniforms is None:
            uniforms = torch.rand(batch_size, dtype=torch.float64, device=self.device, generator=generator)
        u = uniforms.to(self.device, torch.float64).contiguous()
        idxs = torch.empty(batch_size, dtype=torch.int64, device=self.device)
        w32 = torch.empty(batch_size, dtype=torch.float32, device=self.device)
        self._w64 = torch.empty(batch_size, dtype=torch.float64, device=self.device)
        _lib.check(self._L.srl_per_sample(self._h, u.data_ptr(), int(batch_size), float(beta), idxs.data_ptr(), self._w64.data_ptr(), w32.data_ptr(),
                                          self._stream()), 'srl_per_sample')
        return idxs, w32

    def trees(self):
        cap = self.capacity
        s = torch.empty(2 * cap, dtype=torch.float64, device=self.device)
        m = torch.empty(2 * cap, dtype=torch.float64, device=self.device)
        mp = torch.empty(1, dtype=torch.float64, device=self.device)
        _lib.check(self._L.srl_per_debug_trees(self._h, s.data_ptr(), m.data_ptr(), mp.data_ptr(), self._stream()), 'srl_per_debug_trees')
        torch.cuda.current_stream(self.device).synchronize()
        return s, m, float(mp.item())

    def close(self):
        if getattr(self, '_h', None) is not None:
            if self._owned:
                self._L.srl_per_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
