"""Optimizer wrapper with the reference's interface (/root/reference/src/optim.py:5-57) on FLAT fp32 buffers.

All parameters are re-pointed into one contiguous parameter buffer and all gradients into one contiguous gradient
buffer, so that (i) the data-parallel exchange is ONE NCCL all-reduce of `flat_grad`, (ii) the global grad-norm is
one reduction kernel and (iii) clip + NaN-skip + Adadelta/Adam is one fused update kernel that reads the norm on
the device (no host sync in the step, unlike src/solver.py:84-89 which calls math.isnan on a Python float).  The count
of applied steps (torch's state["step"], which a skipped step does not advance) is a device counter for the same
reason: only the device knows whether a step was skipped, also when the step is replayed from a CUDA graph.
"""
from functools import partial

import numpy as np
import torch

from . import lib as L


def speech_aug_scheduler(step, s_r, s_i, s_f, peak_lr):
    """SpecAugment LR schedule (ramp-up / hold / exponential decay to 1%), src/optim.py:59-76."""
    final_ratio = 0.01
    lam = -np.log10(final_ratio) / (s_f - s_i)
    cur = step + 1
    if cur < s_r:
        return peak_lr * float(cur) / s_r
    if cur < s_i:
        return peak_lr
    if cur <= s_f:
        return peak_lr * np.power(10, -lam * (cur - s_i))
    return peak_lr * final_ratio


def _collect(parameters):
    params = []
    for g in parameters:
        if isinstance(g, dict):
            params += list(g["params"])
        else:
            params.append(g)
    return [p for p in params if p.requires_grad]


class FlatBuffers:
    """One contiguous fp32 parameter buffer + one gradient buffer; every nn.Parameter becomes a view."""

    def __init__(self, params):
        self.params = params
        dev = params[0].device
        sizes = [p.numel() for p in params]
        # 16-byte aligned segments so every view can be float4-accessed
        self.offsets = []
        off = 0
        for n in sizes:
            self.offsets.append(off)
            off += (n + 3) // 4 * 4
        self.total = off
        self.flat = torch.zeros(self.total, device=dev, dtype=torch.float32)
        self.grad = torch.zeros(self.total, device=dev, dtype=torch.float32)
        for p, o in zip(params, self.offsets):
            n = p.numel()
            self.flat[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.flat[o:o + n].view(p.shape)
            p.grad = self.grad[o:o + n].view(p.shape)

    def views(self, buf):
        return [buf[o:o + p.numel()].view(p.shape) for p, o in zip(self.params, self.offsets)]

    def rebind_grads(self):
        for p, o in zip(self.params, self.offsets):
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * o:
                g = p.grad
                view = self.grad[o:o + p.numel()].view(p.shape)
                if g is not None:
                    view.copy_(g)
                p.grad = view


class Optimizer:
    """Same constructor / methods as the reference's `Optimizer` (src/optim.py:5-57)."""

    def __init__(self, parameters, optimizer, lr, eps, lr_scheduler, tf_start=1, tf_end=1, tf_step=1, **kwargs):
        self.tf_type = tf_end != 1
        self.tf_rate = lambda step: max(tf_end, tf_start - (tf_start - tf_end) * step / tf_step)
        self.opt_type = optimizer
        self.init_lr = lr
        self.sch_type = lr_scheduler
        self.eps = eps
        self.grad_clip = kwargs.pop("grad_clip", 5.0)
        if optimizer not in ("Adadelta", "Adam"):
            raise NotImplementedError("fused update implemented for Adadelta and Adam (got %s)" % optimizer)
        self.cur_lr = lr
        if lr_scheduler == "warmup":
            warmup_step = 4000.0
            init_lr = lr
            self.lr_scheduler = lambda step: init_lr * warmup_step ** 0.5 * \
                np.minimum((step + 1) * warmup_step ** -1.5, (step + 1) ** -0.5)
            self.cur_lr = 1.0
            self.eps = 1e-6 if optimizer == "Adadelta" else 1e-8   # torch defaults: the reference passes no eps here
        elif lr_scheduler == "spec-aug-basic":
            self.lr_scheduler = partial(speech_aug_scheduler, s_r=500, s_i=20000, s_f=80000, peak_lr=lr)
        elif lr_scheduler == "spec-aug-double":
            self.lr_scheduler = partial(speech_aug_scheduler, s_r=1000, s_i=40000, s_f=160000, peak_lr=lr)
        else:
            self.lr_scheduler = None
        self.rho = 0.9
        self.betas = (0.9, 0.999)
        self.weight_decay = 0.0
        params = _collect(parameters)
        self.buf = FlatBuffers(params)
        dev = self.buf.flat.device
        self.state1 = torch.zeros_like(self.buf.flat)   # Adadelta square_avg / Adam exp_avg
        self.state2 = torch.zeros_like(self.buf.flat)   # Adadelta acc_delta  / Adam exp_avg_sq
        self.step_count = torch.zeros(1, device=dev, dtype=torch.int64)   # applied updates, advanced on the device
        self.grad_norm = torch.zeros(1, device=dev, dtype=torch.float32)
        self._scratch = None
        self.pre_reduce = None    # hook: called with the flat gradient before the norm (data-parallel all-reduce)

    @property
    def n_steps(self):
        """Number of applied updates (steps skipped on a NaN norm excluded); reading it synchronises the device."""
        return int(self.step_count.item())

    # ---- reference API ----
    def get_opt_state_dict(self):
        """torch.optim-shaped state dict (per-parameter views of the flat state)."""
        s1, s2 = self.buf.views(self.state1), self.buf.views(self.state2)
        names = ("square_avg", "acc_delta") if self.opt_type == "Adadelta" else ("exp_avg", "exp_avg_sq")
        state = {}
        n_steps = self.n_steps
        if n_steps > 0:
            for i in range(len(self.buf.params)):
                state[i] = {"step": torch.tensor(float(n_steps)), names[0]: s1[i].clone(), names[1]: s2[i].clone()}
        group = {"lr": self.cur_lr, "eps": self.eps, "weight_decay": self.weight_decay,
                 "params": list(range(len(self.buf.params)))}
        if self.opt_type == "Adadelta":
            group["rho"] = self.rho
        else:
            group["betas"] = self.betas
        return {"state": state, "param_groups": [group]}

    def load_opt_state_dict(self, state_dict):
        names = ("square_avg", "acc_delta") if self.opt_type == "Adadelta" else ("exp_avg", "exp_avg_sq")
        s1, s2 = self.buf.views(self.state1), self.buf.views(self.state2)
        for i, st in state_dict.get("state", {}).items():
            i = int(i)
            s1[i].copy_(st[names[0]])
            s2[i].copy_(st[names[1]])
            if "step" in st:
                self.step_count.fill_(int(float(st["step"])))
        if state_dict.get("param_groups"):
            self.cur_lr = state_dict["param_groups"][0].get("lr", self.cur_lr)

    def pre_step(self, step):
        if self.lr_scheduler is not None:
            self.cur_lr = float(self.lr_scheduler(step))
        self.buf.grad.zero_()
        self.buf.rebind_grads()
        return self.tf_rate(step)

    def step(self):
        """grad-norm + clip(5.0) + NaN skip + update + step count, all on the device; returns the norm (device
        scalar)."""
        lib = L.load()
        b = self.buf
        b.rebind_grads()
        if self.pre_reduce is not None:
            self.pre_reduce(b.grad)
        if self._scratch is None:
            self._scratch = torch.empty(lib.b200asr_grad_norm_scratch_bytes(), dtype=torch.uint8, device=b.flat.device)
        L.check(lib.b200asr_grad_norm(L.ptr(b.grad), b.total, L.ptr(self.grad_norm), L.ptr(self._scratch), L.stream()),
                "grad_norm")
        if self.opt_type == "Adadelta":
            L.check(lib.b200asr_adadelta_step(L.ptr(b.flat), L.ptr(b.grad), L.ptr(self.state1), L.ptr(self.state2),
                                              b.total, self.cur_lr, self.rho, self.eps, self.weight_decay,
                                              L.ptr(self.grad_norm), self.grad_clip, L.ptr(self.step_count),
                                              L.stream()), "adadelta_step")
        else:
            L.check(lib.b200asr_adam_step(L.ptr(b.flat), L.ptr(b.grad), L.ptr(self.state1), L.ptr(self.state2),
                                          b.total, self.cur_lr, self.betas[0], self.betas[1], self.eps,
                                          self.weight_decay, L.ptr(self.grad_norm), self.grad_clip,
                                          L.ptr(self.step_count), L.stream()), "adam_step")
        return self.grad_norm

    def create_msg(self):
        return ["Optim.spec.| Algo. = {}\t| Lr = {}\t (Scheduler = {})| Scheduled sampling = {}".format(
            self.opt_type, self.init_lr, self.sch_type, self.tf_type)]
