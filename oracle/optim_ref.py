"""CPU ORACLE (test infrastructure, NOT a product path) for the fused optimizer step (csrc/optim.cu, optim.Optimizer).

Restates in float64 numpy what the reference does once per training step (src/solver.py:84-89, src/optim.py):
  * clip_grad_norm_(params, 5.0): the 2-norm over every parameter's gradient, coefficient min(1, 5 / (norm + 1e-6));
  * `if math.isnan(norm)` skips optimizer.step(): nothing moves and torch's per-parameter state["step"] does not
    advance.  An Inf norm is not NaN: its coefficient is 5 / inf = 0, so +-Inf gradient entries become NaN, every
    other entry 0, and the step is taken;
  * torch.optim.Adadelta / Adam (L2 weight decay added to the gradient; no amsgrad, maximize or foreach quirks) with
    their constants formed in double as torch forms them: 1 - rho, 1 - beta and the bias corrections 1 - beta ** step
    of the applied-step count.
Pinned against torch.optim on float64 CPU parameters by tests/test_host_optim_oracle.py.
"""
import math

import numpy as np


def grad_norm(grads):
    """Global 2-norm of a list of gradient arrays (NaN if any entry is NaN, Inf if any is +-Inf and none NaN)."""
    return math.sqrt(sum(float(np.sum(np.square(np.asarray(g, np.float64)))) for g in grads))


def clip_coef(norm, max_norm=5.0):
    """clip_grad_norm_'s clamped coefficient; 0 for an Inf norm."""
    return min(1.0, max_norm / (norm + 1e-6))


def clip_grad(g, coef):
    """g times the clip coefficient; +-Inf * 0 = NaN, as in the reference."""
    with np.errstate(invalid="ignore"):
        return np.asarray(g, np.float64) * coef


def adadelta_update(p, g, square_avg, acc_delta, lr=1.0, rho=0.9, eps=1e-6, weight_decay=0.0):
    """One torch.optim.Adadelta update of one parameter, in place on float64 arrays; g already clipped."""
    with np.errstate(invalid="ignore"):
        if weight_decay != 0:
            g = g + weight_decay * p
        square_avg *= rho
        square_avg += (1 - rho) * g * g
        delta = np.sqrt(acc_delta + eps) / np.sqrt(square_avg + eps) * g
        acc_delta *= rho
        acc_delta += (1 - rho) * delta * delta
        p -= lr * delta


def adam_update(p, g, exp_avg, exp_avg_sq, step, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
    """One torch.optim.Adam update of one parameter at applied-step count `step` (>= 1), in place on float64
    arrays; g already clipped."""
    b1, b2 = betas
    with np.errstate(invalid="ignore"):
        if weight_decay != 0:
            g = g + weight_decay * p
        exp_avg *= b1
        exp_avg += (1 - b1) * g
        exp_avg_sq *= b2
        exp_avg_sq += (1 - b2) * g * g
        bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
        p -= lr / bc1 * exp_avg / (np.sqrt(exp_avg_sq / bc2) + eps)


class Optimizer:
    """The reference's step rule over a list of float64 parameter arrays: norm, NaN skip, clip, update."""

    def __init__(self, params, kind, lr, eps, rho=0.9, betas=(0.9, 0.999), weight_decay=0.0, max_norm=5.0):
        if kind not in ("Adadelta", "Adam"):
            raise ValueError(kind)
        self.kind, self.lr, self.eps, self.rho, self.betas = kind, lr, eps, rho, betas
        self.weight_decay, self.max_norm = weight_decay, max_norm
        self.params = [np.array(p, np.float64) for p in params]
        self.state1 = [np.zeros_like(p) for p in self.params]    # square_avg / exp_avg
        self.state2 = [np.zeros_like(p) for p in self.params]    # acc_delta / exp_avg_sq
        self.n_steps = 0                                         # applied updates: torch's state["step"]

    def step(self, grads):
        """-> (norm, applied)."""
        norm = grad_norm(grads)
        if math.isnan(norm):
            return norm, False
        coef = clip_coef(norm, self.max_norm)
        self.n_steps += 1
        for p, g, s1, s2 in zip(self.params, grads, self.state1, self.state2):
            g = clip_grad(g, coef)
            if self.kind == "Adadelta":
                adadelta_update(p, g, s1, s2, self.lr, self.rho, self.eps, self.weight_decay)
            else:
                adam_update(p, g, s1, s2, self.n_steps, self.lr, self.betas, self.eps, self.weight_decay)
        return norm, True
