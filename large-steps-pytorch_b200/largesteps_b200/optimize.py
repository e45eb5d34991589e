"""AdamUniform -- same surface as the reference's largesteps/optimize.py, fused on the GPU.

Variant of Adam with uniform scaling by the second moment: instead of dividing each component by the square root of
its second moment, all of them are divided by the max (optimize.py:3-41).  The reference spends ~8 eager kernels and a
max-reduction per parameter per step; here one step updates every parameter of every group with two kernels per device
(csrc/ls_adam.cu, ls_adam_uniform_step_multi), each parameter still scaled by the max of its own second moment.
"""
import ctypes

import numpy as np
import torch

from . import _native as N


class AdamUniform(torch.optim.Optimizer):
    def __init__(self, params, lr=0.1, betas=(0.9, 0.999)):
        defaults = dict(lr=lr, betas=betas)
        super(AdamUniform, self).__init__(params, defaults)

    def __setstate__(self, state):
        super(AdamUniform, self).__setstate__(state)

    def _scratch(self, dev, n):
        """One device buffer of >= 8 n bytes per device, reused across steps (the callee clears it)."""
        cache = self.__dict__.setdefault("_scratch_by_device", {})
        buf = cache.get(dev)
        if buf is None or buf.numel() < 8 * n:
            buf = cache[dev] = torch.empty(8 * max(n, 16), dtype=torch.uint8, device=dev)
        return buf

    @torch.no_grad()
    def step(self):
        # every parameter is checked before any is updated
        work = []
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    raise RuntimeError("AdamUniform.step(): parameter without gradient (the reference dereferences p.grad too)")
                N.require_cuda(p, "parameter")
                if p.dtype != torch.float32 or not p.data.is_contiguous():
                    raise TypeError("AdamUniform (CUDA) needs contiguous float32 parameters")
                grad = p.grad.data
                if grad.dtype != torch.float32 or grad.device != p.device:
                    raise TypeError("gradient must be float32 on the parameter's device")
                work.append((group, p, grad))
        rows = {}      # device -> table rows of ls_adam_uniform_step_multi
        keep = []      # contiguous copies of non-contiguous gradients, alive until their call is enqueued
        for group, p, grad in work:
            state = self.state[p]
            if len(state) == 0:           # lazy initialization (optimize.py:24-28)
                state["step"] = 0
                state["g1"] = torch.zeros_like(p.data)
                state["g2"] = torch.zeros_like(p.data)
            state["step"] += 1
            if p.numel() == 0:
                continue
            t = state["step"]
            b1, b2 = group['betas']
            grad = grad.contiguous()
            keep.append(grad)
            rows.setdefault(p.device, []).append((
                p.data.data_ptr(), grad.data_ptr(), state["g1"].data_ptr(), state["g2"].data_ptr(), p.numel(),
                float(group['lr']), float(b1), float(b2), float(1 - b1), float(1 - b2),
                float(1 - (b1 ** t)), float(1 - (b2 ** t))))
        lib = N.lib()
        for dev, r in rows.items():
            table = np.array(r, dtype=N.ADAM_TENSOR)
            scratch = self._scratch(dev, len(r))
            with torch.cuda.device(dev):
                N.check(lib.ls_adam_uniform_step_multi(ctypes.c_void_p(table.ctypes.data), len(r), N.ptr(scratch),
                                                       scratch.numel(), N.stream_ptr(dev)), "ls_adam_uniform_step_multi")
