"""Flat parameter / gradient / optimizer-state buffers for the data-parallel step.

The reference keeps per-tensor bf16 params + grads, copies grads into a flat all-reduce buffer and back
(fairseq/distributed/legacy_distributed_data_parallel.py:127-163) and again into flat fp32 master grads
(fairseq/optim/fp16_optimizer.py:109-145).  Here there is ONE layout shared by
    p16  bf16  -- the model's parameters are views of it (state_dict keys unchanged),
    g32  fp32  -- kernels write/accumulate gradients straight into it; NCCL all-reduces it in place;
                  a small tail carries the logging scalars (sample_size, ntokens, ...) through the same
                  all-reduce (SURVEY.md §0.6),
    p32/m/v fp32 -- master weights and Adam moments,
so the update is: backward -> one all-reduce -> esp_sumsq_f32 -> esp_adam_step.  No flatten/unflatten copies.
"""
from collections import OrderedDict

import torch

TAIL = 8  # fp32 slots after the gradients: [sample_size, ntokens, nsentences, loss, nll/aux, 3 spare]
ALIGN = 64  # elements; keeps every tensor 128-byte aligned in both the bf16 and fp32 buffers


class FlatParams:
    def __init__(self, module: torch.nn.Module, groups=(), device=None, channels_last=()):
        """Re-home every parameter of `module` into one flat bf16 buffer.

        groups: iterable of name lists that must be laid out back to back (e.g. q/k/v projection weights,
        so that the fused [3d, d] view is free)."""
        named = OrderedDict(module.named_parameters())
        order, seen = [], set()
        first_of = {g[0]: list(g) for g in groups}
        in_group = {n for g in groups for n in g}
        for n in named:
            if n in seen:
                continue
            if n in first_of:
                for gname in first_of[n]:
                    order.append(gname)
                    seen.add(gname)
            elif n in in_group:
                continue  # emitted with its group head
            else:
                order.append(n)
                seen.add(n)
        assert set(order) == set(named), "parameter groups must be made of existing parameter names"
        self.names = order
        self.offsets, self.shapes = {}, {}
        off = 0
        grouped_next = set()
        for g in groups:
            grouped_next.update(g[:-1])  # no padding after these: the next member must be adjacent
        for n in order:
            p = named[n]
            self.offsets[n] = off
            self.shapes[n] = tuple(p.shape)
            off += p.numel()
            if n not in grouped_next:
                off = (off + ALIGN - 1) // ALIGN * ALIGN
        self.numel = off
        dev = device if device is not None else next(module.parameters()).device
        self.p16 = torch.zeros(self.numel, dtype=torch.bfloat16, device=dev)
        self.g32 = torch.zeros(self.numel + TAIL, dtype=torch.float32, device=dev)
        self.p32 = None  # allocated lazily by the optimizer
        # 4-D conv weights listed in `channels_last` keep their logical [O, I, kh, kw] shape (state_dict unchanged)
        # but are stored O,kh,kw,I in the flat buffers, so cuDNN runs NHWC kernels without layout transposes.
        self.channels_last = set(channels_last)
        for n in order:
            p = named[n]
            view = self._view(self.p16, n)
            view.copy_(p.data.to(device=dev, dtype=torch.bfloat16))
            p.data = view
        self.module = module

    # ---- views --------------------------------------------------------------------------------
    def _view(self, buf, name):
        o, s = self.offsets[name], self.shapes[name]
        n = 1
        for d in s:
            n *= d
        flat = buf[o: o + n]
        if name in self.channels_last and len(s) == 4:
            return flat.view(s[0], s[2], s[3], s[1]).permute(0, 3, 1, 2)
        return flat.view(s)

    def param(self, name):
        return self._view(self.p16, name)

    def grad(self, name):
        return self._view(self.g32, name)

    def span(self, buf, names, shape):
        """One view covering adjacent parameters (asserts adjacency)."""
        o = self.offsets[names[0]]
        n = 0
        for nm in names:
            assert self.offsets[nm] == o + n, "parameters %s are not adjacent in the flat layout" % (names,)
            k = 1
            for d in self.shapes[nm]:
                k *= d
            n += k
        return buf[o: o + n].view(shape)

    @property
    def grads(self):
        return self.g32[: self.numel]

    @property
    def tail(self):
        return self.g32[self.numel:]

    def zero_grad(self):
        self.g32.zero_()

    def fold_torch_grads_(self, module, prefix=""):
        """Add the .grad that autograd left on `module`'s parameters (layers torch executes) into the fp32 gradients and
        clear it; a parameter named n in `module` is prefix + n here."""
        for n, p in module.named_parameters():
            if p.grad is not None:
                self.grad(prefix + n).add_(p.grad.float())
                p.grad = None

    def init_master(self):
        if self.p32 is None:
            self.p32 = self.p16.float()
            self.m = torch.zeros_like(self.p32)
            self.v = torch.zeros_like(self.p32)

    def sync_master_from_model(self):
        """After load_state_dict: master weights follow the (bf16) model parameters."""
        if self.p32 is not None:
            self.p32.copy_(self.p16.float())
