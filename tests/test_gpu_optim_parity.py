"""The fused optimizer step (csrc/optim.cu: global norm, clip, NaN skip, Adadelta / Adam, applied-step count) against
the float64 oracle oracle/optim_ref.py, and optim.Optimizer against torch.optim.Adam under the reference's solver rule.

One-step bounds.  Before each update the device's fp32 (p, g, state, count) is copied to the host and the oracle runs
on it in float64, so each check covers exactly one update.  u = 2^-24, the fp32 unit roundoff; every rounding
(of an operation, or of a constant such as fl(rho), fl(1 - rho), fl(lr), fl(eps), fl(wd)) is <= u relative.  Exact
values are capitals.  The bounds are fixed here, independent of any run; fused multiply-adds only drop roundings.
  norm   fp64 sum of squares (<= n.2^-53 relative), one rounding to fp32:   |nrm - N| <= 1.01u.N, checked at 2u.N
  coef   c = min(1, 5 / (nrm + 1e-6f)): two roundings on top of nrm's:    <= 3.2u.c
  g      G = c.g + wd.p:                 e_G = 4.2u.|c.g| + [wd != 0].u.(|wd.p| + |G|)
Adadelta (all of square_avg, acc_delta non-negative, so for wd = 0 these are relative bounds, 13.4u on square_avg):
  square_avg  S = rho.sq + (1-rho).G^2    e_S = 2u.rho.sq + (1-rho).(3u.G^2 + 2|G|.e_G + e_G^2) + u.S
  delta       Q = sqrt(a + eps) / sqrt(S + eps), D = Q.G:
              sqrt(a + eps) <= 2u relative; sqrt(S + eps) <= e/(sqrt(x) + sqrt(x - e)) + u for x = S + eps,
              e = e_S + u.eps + u.x; r_Q = 2u + r_den / (1 - r_den) + u;   e_D = Q.e_G + |G|.Q.r_Q.(1 + e_G/|G|) + u.|D|
  acc_delta   e_A = 2u.rho.a + (1-rho).(3u.D^2 + 2|D|.e_D + e_D^2) + u.A'
  param       e_P = lr.(e_D + 2u.|D|) + u.|P'|
Adam (step t = the advanced count; bias corrections b1 = 1 - beta1^t, b2 = 1 - beta2^t in double):
  exp_avg     e_M = 2u.beta1.|m| + (1-beta1).(2u.|G| + e_G) + u.|M'|   (7.2u.(beta1.|m| + (1-beta1).|g|) for wd = 0)
  exp_avg_sq  e_V = 2u.beta2.v + (1-beta2).(3u.G^2 + 2|G|.e_G + e_G^2) + u.V'   (13.4u relative for wd = 0)
  denom       X = sqrt(V'/b2) + eps: sqrt(v) as above, times fl(1/sqrt(b2)) (2u), + eps (2u on eps, u on X)
  param       P' = p - fl(lr/b1).(M'/X): e_P = (lr/b1).((|M'| + e_M)/X . r_X/(1 - r_X) + e_M/X + 4u.|M'/X|) + u.|P'|
A few subnormal ulps are added to each bound for the states near 1e-30.  The fp32 complement 1.f - 0.999f is
216u off fl(1 - 0.999), far outside e_V; a bias correction of the wrong step count is off by percent.
"""
import math

import numpy as np
import pytest
import torch

from oracle import optim_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
TINY = 4 * 2.0 ** -149
SIZES = [1, 3, 4, 5, 1027, 100003, 2 ** 22 + 3]     # tail only; tail + float4 body; grid-stride loop
HP = {"Adadelta": dict(lr=1.0, rho=0.9, eps=1e-8), "Adam": dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8)}


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


# ------------------------------------------------------------------------------------------- bounds
def _sqrt_err(x, e):
    """Bound on |sqrt(x') - sqrt(x)| for |x' - x| <= e, x >= 0 (0 where e = 0)."""
    den = np.sqrt(x) + np.sqrt(np.maximum(x - e, 0.0))
    return np.divide(e, den, out=np.zeros_like(e), where=e > 0)


def _grad_err(g, p, coef, wd):
    G = coef * g + wd * p
    e = 4.2 * U * np.abs(coef * g)
    if wd != 0:
        e = e + U * (np.abs(wd * p) + np.abs(G))
    return G, e


def _ema_sq_err(beta, v, G, eG, V):
    """Error of fl(fl(beta).v + fl(1-beta).gi.gi) against V = beta.v + (1-beta).G^2."""
    return 2 * U * beta * v + (1 - beta) * (3 * U * G * G + 2 * np.abs(G) * eG + eG * eG) + U * V


def _rel_inv(r):
    return np.where(r < 1, r / np.maximum(1 - r, 1e-300), np.inf)


def adadelta_bounds(p, g, sq, acc, coef, lr, rho, eps, wd):
    """-> per-element bounds on (square_avg, acc_delta, param) after one update (see the module docstring)."""
    G, eG = _grad_err(g, p, coef, wd)
    S = rho * sq + (1 - rho) * G * G
    eS = _ema_sq_err(rho, sq, G, eG, S)
    x = S + eps
    den = np.sqrt(x)
    r_den = (_sqrt_err(x, eS + U * eps + U * x) + U * den) / den
    Q = np.sqrt(acc + eps) / den
    rQ = 2 * U + _rel_inv(r_den) + U
    D = Q * G
    eD = Q * eG + (np.abs(G) + eG) * Q * rQ + U * np.abs(D)
    A = rho * acc + (1 - rho) * D * D
    eA = _ema_sq_err(rho, acc, D, eD, A)
    P = p - lr * D
    eP = lr * (eD + 2 * U * np.abs(D)) + U * np.abs(P)
    return eS + TINY, eA + TINY, eP + TINY


def adam_bounds(p, g, m, v, t, coef, lr, betas, eps, wd):
    """-> per-element bounds on (exp_avg, exp_avg_sq, param) after one update at step t (see the module docstring)."""
    b1, b2 = betas
    G, eG = _grad_err(g, p, coef, wd)
    M = b1 * m + (1 - b1) * G
    eM = 2 * U * b1 * np.abs(m) + (1 - b1) * (2 * U * np.abs(G) + eG) + U * np.abs(M)
    V = b2 * v + (1 - b2) * G * G
    eV = _ema_sq_err(b2, v, G, eG, V)
    r2 = 1 / math.sqrt(1 - b2 ** t)
    sv = np.sqrt(V)
    X = sv * r2 + eps
    eX = r2 * (_sqrt_err(V, eV) + 3 * U * sv) + 2 * U * eps + U * X
    rX = _rel_inv(eX / X)
    ss = lr / (1 - b1 ** t)
    P = p - ss * M / X
    eP = ss * ((np.abs(M) + eM) / X * rX + eM / X + 4 * U * np.abs(M) / X) + U * np.abs(P)
    return eM + TINY, eV + TINY, eP + TINY


# ------------------------------------------------------------------------------------------- C ABI
class Flat:
    """One flat buffer set on the device, driven through the C ABI as optim.Optimizer drives it."""

    def __init__(self, pkg, kind, n, wd, seed):
        self.L, self.lib = pkg.lib, pkg.lib.load()
        self.kind, self.n, self.wd = kind, n, wd
        self.gen = torch.Generator().manual_seed(seed)
        self.p = torch.randn(n, generator=self.gen).to(DEV)
        self.g = torch.zeros(n, device=DEV)
        self.s1 = torch.zeros(n, device=DEV)
        self.s2 = torch.zeros(n, device=DEV)
        self.count = torch.zeros(1, dtype=torch.int64, device=DEV)
        self.norm = torch.zeros(1, device=DEV)
        self.scratch = torch.empty(self.lib.b200asr_grad_norm_scratch_bytes(), dtype=torch.uint8, device=DEV)

    def host(self):
        return {k: getattr(self, k).cpu().double().numpy() for k in ("p", "g", "s1", "s2")} | \
            {"count": int(self.count.item())}

    def grad_norm(self):
        L = self.L
        L.check(self.lib.b200asr_grad_norm(L.ptr(self.g), self.n, L.ptr(self.norm), L.ptr(self.scratch), L.stream()))
        return self.norm

    def update(self):
        L, h = self.L, HP[self.kind]
        a = (L.ptr(self.p), L.ptr(self.g), L.ptr(self.s1), L.ptr(self.s2), self.n)
        if self.kind == "Adadelta":
            rc = self.lib.b200asr_adadelta_step(*a, h["lr"], h["rho"], h["eps"], self.wd, L.ptr(self.norm), 5.0,
                                                L.ptr(self.count), L.stream())
        else:
            rc = self.lib.b200asr_adam_step(*a, h["lr"], h["betas"][0], h["betas"][1], h["eps"], self.wd,
                                            L.ptr(self.norm), 5.0, L.ptr(self.count), L.stream())
        L.check(rc, self.kind)

    def step(self):
        """norm + update; -> (host copy before, host copy after)."""
        before = self.host()
        self.grad_norm()
        self.update()
        return before, self.host()


def _oracle_and_bounds(kind, h, wd):
    """The oracle's update of the host copy h (dict of float64 arrays) and the per-element bounds."""
    hp = HP[kind]
    norm = optim_ref.grad_norm([h["g"]])
    coef = optim_ref.clip_coef(norm)
    g = optim_ref.clip_grad(h["g"], coef)
    p, s1, s2 = h["p"].copy(), h["s1"].copy(), h["s2"].copy()
    t = h["count"] + 1
    gb = np.where(np.isinf(h["g"]), 0.0, h["g"])
    if kind == "Adadelta":
        optim_ref.adadelta_update(p, g, s1, s2, hp["lr"], hp["rho"], hp["eps"], wd)
        bounds = adadelta_bounds(h["p"], gb, h["s1"], h["s2"], coef, hp["lr"], hp["rho"], hp["eps"], wd)
    else:
        optim_ref.adam_update(p, g, s1, s2, t, hp["lr"], hp["betas"], hp["eps"], wd)
        bounds = adam_bounds(h["p"], gb, h["s1"], h["s2"], t, coef, hp["lr"], hp["betas"], hp["eps"], wd)
    return norm, {"s1": s1, "s2": s2, "p": p}, dict(zip(("s1", "s2", "p"), bounds))


def _check_update(kind, before, after, wd, what):
    norm, ref, bound = _oracle_and_bounds(kind, before, wd)
    assert after["count"] == before["count"] + 1, what
    for k in ("s1", "s2", "p"):
        got, want = after[k], ref[k]
        assert np.array_equal(np.isnan(got), np.isnan(want)), (what, k)
        ok = ~np.isnan(want)
        err = np.abs(got[ok] - want[ok])
        worst = int(np.argmax(err / bound[k][ok]))
        assert np.all(err <= bound[k][ok]), (what, k, float(err[worst] / U), float(bound[k][ok][worst] / U),
                                             float(want[ok][worst]))
    return norm


def _set_grad(f, norm):
    """A random gradient rescaled to the given global norm (0: all zero)."""
    g = torch.randn(f.n, generator=f.gen, dtype=torch.float64)
    f.g.copy_((g * (norm / float(g.norm()))).float() if norm else torch.zeros(f.n))


def _log_uniform(f, lo, hi, signed):
    x = torch.exp(torch.empty(f.n, dtype=torch.float64).uniform_(math.log(lo), math.log(hi), generator=f.gen))
    if signed:
        x = x * torch.where(torch.rand(f.n, generator=f.gen) < 0.5, -1.0, 1.0).double()
    return x.float().to(DEV)


@pytest.mark.parametrize("wd", [0.0, 1e-2])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["Adadelta", "Adam"])
def test_one_step_matches_float64(pkg, kind, n, wd):
    """Regimes in sequence on one buffer set: norm below the clip, far above it, an all-zero gradient, then states
    spread over 1e-30 .. 1e4 (Adam: from step 3000 on, exp_avg of both signs)."""
    f = Flat(pkg, kind, n, wd, seed=n % 1000 + (7 if wd else 0) + (100 if kind == "Adam" else 0))
    for what, norm in (("below", 0.8), ("above", 40.0), ("zero", 0.0), ("states", 40.0), ("states", 3.0)):
        if what == "states":
            f.s1.copy_(_log_uniform(f, 1e-30, 1e4, signed=kind == "Adam"))
            f.s2.copy_(_log_uniform(f, 1e-30, 1e4, signed=False))
            if kind == "Adam" and f.count.item() < 100:
                f.count.fill_(2999)
        _set_grad(f, norm)
        before, after = f.step()
        ref_norm = _check_update(kind, before, after, wd, what)
        got = f.norm.item()
        assert abs(got - ref_norm) <= 2 * U * ref_norm, (what, got, ref_norm)
        first = _bits(f.norm)
        assert torch.equal(_bits(f.grad_norm()), first)           # the same reduction order every run


@pytest.mark.parametrize("kind", ["Adadelta", "Adam"])
@pytest.mark.parametrize("n", [5, 1027])
def test_skip_rules(pkg, kind, n):
    """One NaN entry: nothing moves and the count stays.  One +Inf or -Inf entry: the norm is Inf, the coefficient 0,
    the step is applied and counted, NaN exactly at that entry.  NaN and Inf together: skip."""
    f = Flat(pkg, kind, n, 0.0, seed=11)
    _set_grad(f, 40.0)
    f.step()                                                 # a normal step first: non-zero states
    for what, entries in (("+inf", {n // 2: math.inf}), ("nan", {n - 1: math.nan}), ("-inf", {0: -math.inf}),
                          ("nan+inf", {1: math.nan, n - 2: math.inf})):
        _set_grad(f, 40.0)
        for i, x in entries.items():
            f.g[i] = x
        state = [_bits(t) for t in (f.p, f.s1, f.s2)]
        before, after = f.step()
        if math.isnan(f.norm.item()):
            assert what in ("nan", "nan+inf"), what
            assert after["count"] == before["count"], what
            for a, t in zip(state, (f.p, f.s1, f.s2)):
                assert torch.equal(a, _bits(t)), what
        else:
            assert what in ("+inf", "-inf") and math.isinf(f.norm.item()), what
            _check_update(kind, before, after, 0.0, what)
            bad = next(iter(entries))
            assert np.flatnonzero(np.isnan(after["p"])).tolist() == [bad], what
            f.p[bad] = 0.0                                   # keep the next step's parameters finite
            f.s1[bad] = 0.0
            f.s2[bad] = 0.0


# ------------------------------------------------------------------------------------------- Optimizer
SHAPES = [(3,), (5, 7), (11,), (2, 3, 3), (1,)]            # no size a multiple of 4: every segment is padded


def _adam_pair(pkg, seed):
    g = torch.Generator().manual_seed(seed)
    host = [torch.randn(s, generator=g) for s in SHAPES]
    mine = [torch.nn.Parameter(h.to(DEV)) for h in host]
    opt = pkg.Optimizer([{"params": mine}], "Adam", 1e-3, 1e-8, "fixed")
    ref = [torch.nn.Parameter(h.clone()) for h in host]
    return mine, opt, ref, torch.optim.Adam(ref, lr=1e-3, betas=(0.9, 0.999), eps=1e-8)


def _both_step(mine, opt, ref, ref_opt, grads, step):
    """Our Optimizer step and the reference's solver rule on torch.optim (src/solver.py:84-89)."""
    opt.pre_step(step)
    for p, g in zip(mine, grads):
        p.grad.copy_(g.to(DEV))
    opt.step()
    for p, g in zip(ref, grads):
        p.grad = g.clone()
    norm = torch.nn.utils.clip_grad_norm_(ref, 5.0)
    if not math.isnan(norm):
        ref_opt.step()


def _ref_count(ref_opt):
    st = ref_opt.state_dict()["state"]
    return int(float(st[0]["step"])) if st else 0


def _assert_same(mine, opt, ref, ref_opt, applied, what):
    """fp32 on both sides, each update within a few tens of u of fp64: 1e-4 lr per applied update is generous, and
    the bias corrections of a wrong step count are off by 25 % of lr at the first update after a skip."""
    assert opt.n_steps == _ref_count(ref_opt) == applied, what
    for a, b in zip(mine, ref):
        d = (a.detach().cpu() - b.detach()).abs()
        assert float((d - 16 * U * b.detach().abs()).max()) <= 1e-4 * 1e-3 * max(applied, 1), what
    buf = opt.buf
    pad = torch.ones(buf.total, dtype=torch.bool, device=DEV)
    for p, o in zip(buf.params, buf.offsets):
        pad[o:o + p.numel()] = False
    assert int(pad.sum()) > 0
    for t in (buf.flat, opt.state1, opt.state2):             # the padding of the flat buffers stays exactly 0
        assert torch.equal(_bits(t[pad]), torch.zeros(int(pad.sum()), dtype=torch.int32)), what


def _grads(g, kind):
    out = [torch.randn(s, generator=g) * 3 for s in SHAPES]
    if kind == "skip":
        out[3][1, 2, 0] = math.nan
    return out


def test_adam_through_optimizer_counts_applied_steps_and_round_trips(pkg):
    """skip, apply, apply, skip, apply against torch.optim.Adam; then get_opt_state_dict() loaded into torch.optim.Adam
    and torch's state_dict() loaded with load_opt_state_dict() both continue as the original pair does."""
    mine, opt, ref, ref_opt = _adam_pair(pkg, seed=21)
    g = torch.Generator().manual_seed(22)
    applied = 0
    for i, what in enumerate(("skip", "apply", "apply", "skip", "apply")):
        _both_step(mine, opt, ref, ref_opt, _grads(g, what), i)
        applied += what == "apply"
        _assert_same(mine, opt, ref, ref_opt, applied, "%d %s" % (i, what))

    # ours -> torch
    ours_sd = opt.get_opt_state_dict()
    t2 = [torch.nn.Parameter(p.detach().cpu().clone()) for p in mine]
    t2_opt = torch.optim.Adam(t2, lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    t2_opt.load_state_dict(ours_sd)
    # torch -> ours
    m2 = [torch.nn.Parameter(p.detach().clone().to(DEV)) for p in ref]
    m2_opt = pkg.Optimizer([{"params": m2}], "Adam", 1e-3, 1e-8, "fixed")
    m2_opt.load_opt_state_dict(ref_opt.state_dict())
    assert m2_opt.n_steps == applied
    for i, what in enumerate(("apply", "skip", "apply"), start=5):
        grads = _grads(g, what)
        _both_step(mine, opt, t2, t2_opt, grads, i)
        _both_step(m2, m2_opt, ref, ref_opt, grads, i)
        applied += what == "apply"
        _assert_same(mine, opt, t2, t2_opt, applied, "ours -> torch, %d %s" % (i, what))
        _assert_same(m2, m2_opt, ref, ref_opt, applied, "torch -> ours, %d %s" % (i, what))
    assert float(opt.get_opt_state_dict()["state"][0]["step"]) == applied


# ------------------------------------------------------------------------------------------- CUDA graph
def test_replayed_adadelta_steps_count_only_applied_updates(pkg):
    """A captured Adadelta TrainStep: the checkpoint's step is the number of applied updates, eager and replayed; the
    replay on an infeasible batch (NaN norm) does not count, and the capture itself applies nothing."""
    from test_gpu_kernel_variants import LONG_TEXT, _skip_batch
    from test_gpu_model import _tiny_config
    _, _, batch, txt = _skip_batch([9000, 9000, 9000], LONG_TEXT)
    wave, txt = batch.to(DEV), txt.to(DEV)
    full, cut = torch.tensor([9000, 9000, 9000]), torch.tensor([9000, 9000, 6400])
    step = pkg.TrainStep(_tiny_config("hybrid"), 12, device=DEV, seed=5)
    assert step.capture(wave, full, txt, warmup=3), step.graph_error
    opt = step.optimizer
    assert opt.n_steps == 3                                   # the eager warm-up steps
    applied = 3
    for lens in (full, cut, full, full):
        step(wave, lens, txt)
        assert step.graph is not None
        applied += not math.isnan(opt.grad_norm.item())
        assert opt.n_steps == applied
    assert applied == 6
    sd = opt.get_opt_state_dict()
    assert sd["state"] and all(float(s["step"]) == applied for s in sd["state"].values())
