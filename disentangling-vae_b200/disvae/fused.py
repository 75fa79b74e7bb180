"""Optimizer step and whole-step CUDA-graph capture for the Trainer (SURVEY.md section 8f-2).

`FusedAdam` drives `dv_adam_multi` (one launch for every parameter tensor of a model) with the
hyper-parameters and the state dictionary of the `torch.optim.Adam` instance that `main.py`
constructed (main.py:208, losses.py:238): `optimizer.state[p]` holds the very buffers the kernel
updates, so `optimizer.state_dict()` stays meaningful (the step
counter is mirrored back by `flush_state`, which the Trainer calls at every epoch end).  Anything other than a plain Adam (amsgrad,
weight decay, maximize, non-CUDA parameters) is not taken over: `FusedAdam.supports` says no and the
caller keeps using `optimizer.step()`.
"""
import ctypes

import torch

from . import _native as N


class FusedAdam:
    @staticmethod
    def supports(optimizer):
        if type(optimizer) is not torch.optim.Adam:
            return False
        n = 0
        for g in optimizer.param_groups:
            if g.get("amsgrad") or g.get("weight_decay", 0) != 0 or g.get("maximize") or g.get("differentiable"):
                return False
            for p in g["params"]:
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    return False
                n += 1
        return 0 < n

    @staticmethod
    def lazy(holder, attr, optimizer):
        """`holder.<attr>`: the FusedAdam over `optimizer`, built at the first call (once the parameters are on the
        device); False where `supports` says no, and the caller keeps `optimizer.step()`."""
        fused = getattr(holder, attr)
        if fused is None:
            fused = FusedAdam(optimizer) if FusedAdam.supports(optimizer) else False
            setattr(holder, attr, fused)
        return fused

    def __init__(self, optimizer):
        assert FusedAdam.supports(optimizer)
        self.optimizer = optimizer
        self.max_tensors = N.lib().dv_adam_multi_max_tensors()
        self.host_steps = 0
        self.groups = []
        for g in optimizer.param_groups:
            params = [p for p in g["params"] if p.requires_grad]
            step0 = 0.0
            for p in params:
                st = optimizer.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                step0 = float(st["step"])
            self.groups.append(dict(group=g, params=params, step0=step0,
                                    step_dev=torch.full((1,), step0, dtype=torch.float32, device=params[0].device)))

    def step(self, grad_scale=1.0):
        """One Adam update of every parameter that has a gradient (torch.optim.Adam semantics)."""
        for G in self.groups:
            g = G["group"]
            live = [p for p in G["params"] if p.grad is not None]
            for i in range(0, len(live), self.max_tensors):
                chunk = live[i:i + self.max_tensors]
                n = len(chunk)
                arr = ctypes.c_void_p * n
                st = [self.optimizer.state[p] for p in chunk]
                grads = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in chunk]
                N.call("dv_adam_multi", n, arr(*[p.data_ptr() for p in chunk]), arr(*[t.data_ptr() for t in grads]),
                       arr(*[s["exp_avg"].data_ptr() for s in st]), arr(*[s["exp_avg_sq"].data_ptr() for s in st]),
                       (ctypes.c_longlong * n)(*[p.numel() for p in chunk]), N.ptr(G["step_dev"]),
                       g["lr"], g["betas"][0], g["betas"][1], g["eps"], grad_scale, N.stream())
                # the kernel advances step_dev once per call; keep chunks of one group on the same step
                if i + self.max_tensors < len(live):
                    G["step_dev"] -= 1.0
        self.host_steps += 1

    def flush_state(self):
        """Write the step counters back into optimizer.state: the count the optimizer was constructed/loaded with
        plus the steps taken here (host mirror of the device counter; no sync).  The Trainer calls this at every
        epoch end, so `optimizer.state_dict()` saved at a checkpoint resumes with the right bias correction."""
        for G in self.groups:
            for p in G["params"]:
                self.optimizer.state[p]["step"].fill_(float(G["step0"] + self.host_steps))
