"""Multi-tensor Adam on one hand-written kernel launch per parameter group (csrc/mg_optim.cu).

Drop-in for the ``torch.optim.Adam(model.parameters(), lr, betas=[b1, b2])`` the reference constructs at
train.py:51-52: same constructor arguments, same update arithmetic (L2 weight decay, no amsgrad), same per-parameter
state keys (``step``, ``exp_avg``, ``exp_avg_sq``), so optimizer checkpoints written by either load into the other
(train.py:27-29,36-37).  The reference's optimizer issues ~10 foreach launches sequences over 90 / 63 tensors per step
per step; here a step is one launch driven by a device-side pointer table that is rebuilt only when
a tensor moved.  CUDA fp32 parameters only.
"""
import ctypes

import torch

from . import engine as _engine


def _bump_versions(params):
    inc = getattr(torch._C, "_increment_version", None)
    if inc is not None:
        try:
            inc(params)  # torch >= 2.4: takes an iterable of tensors
            return
        except TypeError:
            for p in params:
                inc(p)
            return
    for p in params:  # very old torch: a no-op in-place op (one tiny launch per tensor)
        p.add_(0)


class Adam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False):
        if amsgrad:
            raise _engine.EngineError("melgan_multi_b200.optim.Adam: amsgrad is not implemented")
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1 or weight_decay < 0:
            raise ValueError("invalid Adam hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False))
        self._tables = {}

    # -- host side of the launch: everything that does not change between steps is cached ------------------------
    def _table(self, gi, ps):
        """Device-side tables of one group.  Parameter / moment pointers, sizes and the CTA map are built once (until the
        set of tensors with a gradient changes); only the gradient pointers, which autograd reallocates every step, are
        refreshed: one small pinned-to-device copy."""
        # identity AND storage of every tensor the kernel writes through: after model.to(...), p.data = ..., or a moment
        # replaced outside load_state_dict, a cached raw pointer would be a silent write into freed memory
        ids = tuple((id(p), p.data_ptr(), self.state[p]["exp_avg"].data_ptr(), self.state[p]["exp_avg_sq"].data_ptr()) for p in ps)
        tab = self._tables.get(gi)
        if tab is None or tab["ids"] != ids:
            if tab is not None:
                self._flush_steps(gi)  # the old table's step count goes back into state before it is replaced
            dev = ps[0].device
            chunk = _engine.lib().mg_adam_chunk()
            first, total = [], 0
            for p in ps:
                first.append(total)
                total += (p.numel() + chunk - 1) // chunk
            first.append(total)

            def col(vals, dtype=torch.int64):
                return torch.tensor(vals, dtype=dtype).to(dev)
            tab = dict(ids=ids, count=len(ps), total=total, n=col([p.numel() for p in ps]), first=col(first, torch.int32),
                       p=col([p.data_ptr() for p in ps]), m=col([self.state[p]["exp_avg"].data_ptr() for p in ps]),
                       v=col([self.state[p]["exp_avg_sq"].data_ptr() for p in ps]),
                       g=torch.empty(len(ps), dtype=torch.int64, device=dev),
                       pin=[torch.empty(len(ps), dtype=torch.int64).pin_memory() for _ in range(2)], uploaded=[None, None],
                       flip=0, grads=None)
            self._tables[gi] = tab
        if tab.get("t") is None:
            tab["t"] = self._group_step(ps)  # (re)read the step count from state for a new table
        ptrs = [p.grad.data_ptr() for p in ps]  # (holding the grad tensors to compare identities would keep them alive)
        if ptrs != tab["grads"]:
            # The upload is asynchronous: a pinned buffer may be rewritten only once the copy that read it has run, or a
            # host running steps ahead of the GPU would hand an earlier step's kernel a later step's gradient pointers.
            # Each buffer keeps the event recorded after its last upload; a loop that syncs every step finds it complete.
            i = tab["flip"]
            tab["flip"] ^= 1
            if tab["uploaded"][i] is not None:
                tab["uploaded"][i].synchronize()
            pin = tab["pin"][i]
            pin.copy_(torch.tensor(ptrs, dtype=torch.int64))
            tab["g"].copy_(pin, non_blocking=True)
            ev = tab["uploaded"][i] = tab["uploaded"][i] or torch.cuda.Event()
            ev.record(torch.cuda.current_stream(tab["g"].device))
            tab["grads"] = ptrs
        return tab

    def _group_step(self, ps):
        steps = {int(self.state[p]["step"]) for p in ps}
        if len(steps) != 1:
            raise _engine.EngineError("melgan_multi_b200.optim.Adam: parameters of one group are at different steps")
        return steps.pop()

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        L = _engine.lib()
        for gi, group in enumerate(self.param_groups):
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            dev = ps[0].device
            fresh = [p for p in ps if len(self.state[p]) == 0]
            for p in ps:
                if not p.is_cuda or p.dtype != torch.float32 or p.grad.is_sparse or p.device != dev or not p.is_contiguous():
                    raise _engine.EngineError("melgan_multi_b200.optim.Adam handles dense contiguous fp32 CUDA parameters on one device")
                if not p.grad.is_contiguous():
                    p.grad = p.grad.contiguous()
            for p in fresh:
                st = self.state[p]
                st["step"] = torch.tensor(0.0)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            tab = self._table(gi, ps)
            # the per-parameter `step` tensors (torch.optim.Adam's state format) are only touched when somebody looks:
            # between steps the count lives in one Python int per group
            if fresh:
                tab["t"] = self._group_step(ps)
            tab["t"] += 1
            tab["dirty"] = True
            b1, b2 = group["betas"]
            with torch.cuda.device(dev):
                stream = torch.cuda.current_stream().cuda_stream
                _engine.check(L.mg_adam_step(tab["p"].data_ptr(), tab["g"].data_ptr(), tab["m"].data_ptr(), tab["v"].data_ptr(),
                                             tab["n"].data_ptr(), tab["first"].data_ptr(), tab["count"], tab["total"],
                                             ctypes.c_float(group["lr"]), ctypes.c_float(b1), ctypes.c_float(b2),
                                             ctypes.c_float(group["eps"]), ctypes.c_float(group["weight_decay"]),
                                             ctypes.c_longlong(tab["t"]), stream))
            # The kernel wrote the parameters through raw pointers, which autograd's version counters cannot see.  Everything
            # that caches derived state keyed on ``_version`` -- the modules' packed weight-norm folds (models.py
            # ``_ensure_packed``), autograd's saved-tensor checks -- must observe an in-place update, exactly as after
            # torch.optim.Adam: bump every updated parameter's counter (no kernel, no copy).
            _bump_versions(ps)
        return loss

    def _flush_steps(self, only=None):
        for gi, tab in self._tables.items():
            if (only is None or gi == only) and tab.get("dirty"):
                live = {i[0] for i in tab["ids"]}
                for p in self.param_groups[gi]["params"]:
                    if id(p) in live:
                        self.state[p]["step"] = torch.tensor(float(tab["t"]))
                tab["dirty"] = False

    def state_dict(self):
        self._flush_steps()
        return super().state_dict()

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._tables = {}  # moments were replaced: rebuild the pointer tables and re-read the step counts
