"""Optimizer step and whole-step CUDA-graph capture for the Trainer (SURVEY.md section 8f-2).

`FusedAdam` drives `dv_adam_multi` (one launch for every parameter tensor of a model) with the
hyper-parameters and the state dictionary of the `torch.optim.Adam` instance that `main.py`
constructed (main.py:208, losses.py:238): `optimizer.state[p]` holds the very buffers the kernel
updates, so `optimizer.state_dict()` stays meaningful (the per-parameter step counts are mirrored back by
`flush_state`, which the Trainer calls at every epoch end).  Anything other than a plain Adam (amsgrad,
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
            base = []
            for p in params:
                st = optimizer.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                base.append(float(st["step"]))
            # parameter i has taken base[i] + host_steps steps; step_dev holds dev_base + host_steps
            self.groups.append(dict(group=g, params=params, base=base, dev_base=base[0],
                                    step_dev=torch.full((1,), base[0], dtype=torch.float32, device=params[0].device)))

    def step(self, grad_scale=1.0):
        """One Adam update of every parameter that has a gradient (torch.optim.Adam semantics: a parameter without one
        keeps its state, its step count included, and each parameter's bias correction follows its own count)."""
        for G in self.groups:
            params, base = G["params"], G["base"]
            live = [i for i, p in enumerate(params) if p.grad is not None]
            if len(live) == len(params) and all(b == G["dev_base"] for b in base):
                self._launch(G, params, G["step_dev"], grad_scale)      # the training step: one counter for all
                continue
            # Some parameters skip this step or sit at other step counts: one dv_adam_multi call per distinct count.
            # These are host-side decisions that a CUDA graph replay would not repeat, so they may not be captured.
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("FusedAdam: a captured step must update every parameter of a group at one step "
                                   "count (%d of %d parameters have a gradient)" % (len(live), len(params)))
            counts = sorted({base[i] for i in live})
            if len(counts) == 1 and len(live) == len(params):
                G["step_dev"].fill_(counts[0] + self.host_steps)          # counts equal again: back to one counter
                G["dev_base"] = counts[0]
                self._launch(G, params, G["step_dev"], grad_scale)
                continue
            if counts:
                step_devs = torch.tensor([c + self.host_steps for c in counts], dtype=torch.float32,
                                         device=params[0].device)
                for k, c in enumerate(counts):
                    self._launch(G, [params[i] for i in live if base[i] == c], step_devs[k:k + 1], grad_scale)
            skipped = set(range(len(params))) - set(live)
            for i in skipped:
                base[i] -= 1.0                       # host_steps advances below; a skipped parameter's count does not
            G["dev_base"] -= 1.0                     # nor does step_dev
        self.host_steps += 1

    def _launch(self, G, params, step_dev, grad_scale):
        """dv_adam_multi over `params` (all at the step count `step_dev` holds), max_tensors per call."""
        g = G["group"]
        for i in range(0, len(params), self.max_tensors):
            chunk = params[i:i + self.max_tensors]
            n = len(chunk)
            arr = ctypes.c_void_p * n
            st = [self.optimizer.state[p] for p in chunk]
            grads = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in chunk]
            N.call("dv_adam_multi", n, arr(*[p.data_ptr() for p in chunk]), arr(*[t.data_ptr() for t in grads]),
                   arr(*[s["exp_avg"].data_ptr() for s in st]), arr(*[s["exp_avg_sq"].data_ptr() for s in st]),
                   (ctypes.c_longlong * n)(*[p.numel() for p in chunk]), N.ptr(step_dev),
                   g["lr"], g["betas"][0], g["betas"][1], g["eps"], grad_scale, N.stream())
            # the kernel advances step_dev once per call; keep chunks of one step count on the same step
            if i + self.max_tensors < len(params):
                step_dev -= 1.0

    def flush_state(self):
        """Write the step counts back into optimizer.state: each parameter's count at construction/load plus the steps
        it took here (host mirror of the device counters; no sync).  The Trainer calls this at every epoch end, so
        `optimizer.state_dict()` saved at a checkpoint resumes with the right bias correction."""
        for G in self.groups:
            for p, b in zip(G["params"], G["base"]):
                self.optimizer.state[p]["step"].fill_(float(b + self.host_steps))
