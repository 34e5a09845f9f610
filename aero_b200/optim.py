"""Fused multi-tensor Adam on the CUDA kernels (SURVEY.md section 8f rank 1; reference train.py:83
``torch.optim.Adam(model.parameters(), lr=args.lr, betas=(0.9, args.beta2))``).

``FusedAdam`` is a ``torch.optim.Optimizer``: same constructor arguments, ``state_dict`` keys (``step``, ``exp_avg``,
``exp_avg_sq``) and update rule as ``torch.optim.Adam`` (no amsgrad, no weight decay), but ``step()`` is ONE kernel launch per
parameter group (``aero_adam_step``) over a device table of {param, grad, exp_avg, exp_avg_sq} records instead of a few hundred
small ones.  Parameters of a group whose per-parameter step counts differ (some ``.grad`` was None on earlier steps) get one
launch per distinct count, so that each gets torch's bias correction.
``grad_scale`` multiplies every gradient inside the kernel (1/world_size after a sum all-reduce of a flat gradient buffer)."""
from __future__ import annotations

import ctypes as C
import struct

import torch

from . import cabi

_CHUNK = 1 << 16


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))
        self._tables = {}

    def _table(self, slot, ps):
        """Device chunk table of parameters ps, cached per slot under every pointer it holds: rebuilt when a .grad is re-allocated
        or load_state_dict replaces the moment tensors."""
        key = tuple((p.data_ptr(), p.grad.data_ptr(), self.state[p]["exp_avg"].data_ptr(), self.state[p]["exp_avg_sq"].data_ptr())
                    for p in ps)
        cached = self._tables.get(slot)
        if cached is not None and cached[0] == key:
            return cached
        recs = bytearray()
        n = 0
        for p in ps:
            if p.dtype != torch.float32 or not p.is_cuda or not p.is_contiguous() or not p.grad.is_contiguous():
                raise TypeError("FusedAdam: contiguous fp32 CUDA parameters / gradients only")
            st = self.state[p]
            for off in range(0, p.numel(), _CHUNK):
                cnt = min(_CHUNK, p.numel() - off)
                recs += struct.pack("<QQQQq", p.data_ptr() + 4 * off, p.grad.data_ptr() + 4 * off, st["exp_avg"].data_ptr() + 4 * off,
                                    st["exp_avg_sq"].data_ptr() + 4 * off, cnt)
                n += 1
        dev = ps[0].device
        table = torch.frombuffer(recs, dtype=torch.uint8).clone().to(dev)
        self._tables[slot] = (key, table, n)
        return self._tables[slot]

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = cabi.load()
        used = {}
        for gi, group in enumerate(self.param_groups):
            # torch.optim.Adam counts steps per parameter (a parameter whose .grad was None has taken fewer), and the bias correction
            # follows that count: one launch per distinct count -- a single launch when every parameter has stepped equally often
            by_step = {}
            for i, p in enumerate(group["params"]):
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = torch.zeros((), dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["step"] += 1
                by_step.setdefault(int(st["step"]), []).append(i)
            b1, b2 = group["betas"]
            for step, idx in by_step.items():
                ps = [group["params"][i] for i in idx]
                slot = (gi, tuple(idx))
                _, table, n = used[slot] = self._table(slot, ps)
                with torch.cuda.device(ps[0].device):
                    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                    cabi.check(lib.aero_adam_step(C.c_void_p(table.data_ptr()), n, float(group["lr"]), float(b1), float(b2),
                                                  float(group["eps"]), step, float(grad_scale), stream), lib)
        self._tables = used
        return loss
