"""Gradient hygiene + global-norm clip + Adam / AdamW as two fused launches (csrc/optim_step.cu, SURVEY.md section 8f-3).

`FusedAdam` is a `torch.optim.Optimizer` with torch.optim.Adam's state layout (`step`, `exp_avg`, `exp_avg_sq` per
parameter, so the reference's optimizer checkpoints load) whose `step()` performs what the reference's train loop does
around its optimizer (ca_code/utils/train.py:209-215):

    p.grad[isnan] = 0; p.grad[isinf] = 0;  clip_grad_norm_(params, max_norm);  optimizer.step()

Parameter groups keep their own `lr` / `weight_decay` (the reference's `per_module` learning rates, config/*.yml)."""
import ctypes
import math
import struct
from typing import Optional

import torch

from . import _lib


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, adamw=False,
                 max_grad_norm: Optional[float] = 1.0, sanitize: bool = True, write_clipped_grads: bool = False):
        if lr < 0 or eps < 0 or not (0 <= betas[0] < 1 and 0 <= betas[1] < 1):
            raise ValueError("invalid Adam hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        betas_set = {tuple(g["betas"]) for g in self.param_groups}
        eps_set = {g["eps"] for g in self.param_groups}
        if len(betas_set) != 1 or len(eps_set) != 1:
            raise ValueError("FusedAdam: betas and eps are shared by all groups (lr and weight_decay may differ)")
        self.adamw, self.max_grad_norm, self.sanitize, self.write_clipped_grads = adamw, max_grad_norm, sanitize, write_clipped_grads
        self._table_key = None
        self._table = self._chunks = None
        self._n_chunks = 0
        self._sqnorm = None
        self._steps = 0
        self._missed = {}   # parameter -> number of steps it had no gradient

    # ---- device table of {p, g, m, v, numel, lr, wd} rows + chunk map, rebuilt when a pointer or a rate changes
    def _build(self):
        L = _lib.kernels()
        chunk = L.gb_optim_chunk_elems()
        assert L.gb_optim_row_bytes() == 56
        rows, chunks, key = [], [], []
        dev = None
        for group in self.param_groups:
            for p in group["params"]:
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise RuntimeError("FusedAdam: parameters must be contiguous fp32 CUDA tensors (no CPU fallback)")
                dev = p.device if dev is None else dev
                if p.device != dev:
                    raise RuntimeError("FusedAdam: all parameters on one device")
                st = self.state[p]
                if "exp_avg" not in st:
                    st["step"] = torch.tensor(0.0)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                g = p.grad
                if g is not None and (not g.is_contiguous() or g.dtype != torch.float32):
                    raise RuntimeError("FusedAdam: gradients must be contiguous fp32")
                gp = 0 if g is None else g.data_ptr()
                if g is None:   # torch.optim skips the parameter and does not advance its step count
                    self._missed[p] = self._missed.get(p, 0) + 1
                t = len(rows)
                rows.append(struct.pack("<QQQQqffii", p.data_ptr(), gp, st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                                        p.numel(), float(group["lr"]), float(group["weight_decay"]), self._missed.get(p, 0), 0))
                key.append((p.data_ptr(), gp, p.numel(), float(group["lr"]), float(group["weight_decay"]), self._missed.get(p, 0)))
                for c in range((p.numel() + chunk - 1) // chunk):
                    chunks.append((t, c))
        key = tuple(key)
        if key != self._table_key:
            self._table = torch.frombuffer(bytearray(b"".join(rows)), dtype=torch.uint8).to(dev)
            self._chunks = torch.tensor(chunks, dtype=torch.int32).reshape(-1, 2).to(dev)
            self._n_chunks = len(chunks)
            self._sqnorm = torch.zeros(1, dtype=torch.float64, device=dev)
            self._table_key = key
        return dev

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        dev = self._build()
        if dev is None or self._n_chunks == 0:
            return loss
        L = _lib.kernels()
        self._steps += 1
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is not None:
                    self.state[p]["step"] += 1
        b1, b2 = self.param_groups[0]["betas"]
        t = self._steps
        clip = self.max_grad_norm is not None and self.max_grad_norm > 0
        if self.sanitize or clip:
            self._sqnorm.zero_()
            L.gb_grad_sanitize_sqnorm(self._table, self._chunks, self._n_chunks, self._sqnorm)
        L.gb_adam_step(self._table, self._chunks, self._n_chunks, self._sqnorm if clip else None,
                       float(self.max_grad_norm or 0.0), float(b1), float(b2), float(self.param_groups[0]["eps"]),
                       int(t), int(self.adamw), int(self.write_clipped_grads))
        return loss

    def grad_norm(self) -> torch.Tensor:
        """global L2 norm of the (sanitised) gradients of the last step — a device scalar, no synchronisation"""
        return self._sqnorm.sqrt().float() if self._sqnorm is not None else torch.zeros(())

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        steps = {p: float(st["step"]) for p, st in self.state.items() if "step" in st}
        self._steps = int(max(steps.values())) if steps else 0
        self._missed = {p: self._steps - int(v) for p, v in steps.items() if self._steps - int(v) > 0}
        self._table_key = None
