"""The float64 optimizer oracle (oracle/optim_ref.py) against torch.optim driven by the reference's solver rule
(src/solver.py:84-89: clip_grad_norm_(params, 5.0), then optimizer.step() unless the norm is NaN) on float64 CPU
parameters: scripted gradient sequences over several parameter tensors, with NaN and +-Inf entries, compared in
parameters, optimizer states and state_dict()["state"][i]["step"] after every step."""
import math

import numpy as np
import pytest
import torch

from oracle import optim_ref

SHAPES = [(3,), (4, 5), (7,), (1,)]
NAMES = {"Adadelta": ("square_avg", "acc_delta"), "Adam": ("exp_avg", "exp_avg_sq")}


def _grads(kind, rng):
    """One step's gradients.  'big': norm far above the clip; 'small': below it."""
    scale = {"big": 4.0, "small": 0.05, "zero": 0.0}.get(kind, 1.0)
    gs = [rng.standard_normal(s) * scale for s in SHAPES]
    if kind in ("nan", "nan_inf"):
        gs[1][2, 3] = np.nan
    if kind in ("inf", "nan_inf"):
        gs[0][1] = np.inf
    if kind == "-inf":
        gs[2][6] = -np.inf
    return gs


# skip first (no state yet), Inf steps between applied ones, NaN + Inf together (skip), an all-zero gradient
SEQUENCE = ["nan", "big", "small", "inf", "big", "nan_inf", "zero", "-inf", "small", "nan", "big"]


def _torch_opt(kind, params, wd):
    if kind == "Adadelta":
        return torch.optim.Adadelta(params, lr=1.0, rho=0.9, eps=1e-6, weight_decay=wd)
    return torch.optim.Adam(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)


@pytest.mark.parametrize("kind", ["Adadelta", "Adam"])
@pytest.mark.parametrize("wd", [0.0, 1e-2])
def test_oracle_matches_torch_optim_over_a_sequence(kind, wd):
    rng = np.random.default_rng(7)
    p0 = [rng.standard_normal(s) for s in SHAPES]
    params = [torch.nn.Parameter(torch.from_numpy(p.copy())) for p in p0]
    opt = _torch_opt(kind, params, wd)
    ref = optim_ref.Optimizer(p0, kind, lr=1.0 if kind == "Adadelta" else 1e-3,
                              eps=1e-6 if kind == "Adadelta" else 1e-8, weight_decay=wd)
    applied = 0
    nan_at = [np.zeros(s, bool) for s in SHAPES]      # an applied Inf step leaves NaN at its entries, for good
    for what in SEQUENCE:
        gs = _grads(what, rng)
        for p, g in zip(params, gs):
            p.grad = torch.from_numpy(g.copy())
        tn = float(torch.nn.utils.clip_grad_norm_(params, 5.0))
        if not math.isnan(tn):
            opt.step()
            applied += 1
            nan_at = [m | np.isinf(g) for m, g in zip(nan_at, gs)]
        norm, did = ref.step(gs)
        assert did == (not math.isnan(tn)) and ref.n_steps == applied, what
        assert (math.isnan(norm) and math.isnan(tn)) or norm == tn or abs(norm - tn) <= 1e-14 * tn, what
        state = opt.state_dict()["state"]
        if applied == 0:
            assert state == {}
        for i, p in enumerate(params):
            assert np.array_equal(np.isnan(ref.params[i]), nan_at[i]), what
            np.testing.assert_allclose(p.detach().numpy(), ref.params[i], rtol=1e-12, atol=1e-14, err_msg=what)
            if applied:
                assert float(state[i]["step"]) == ref.n_steps
                for name, mine in zip(NAMES[kind], (ref.state1[i], ref.state2[i])):
                    np.testing.assert_allclose(state[i][name].numpy(), mine, rtol=1e-12, atol=1e-14, err_msg=what)
    assert applied == sum(w not in ("nan", "nan_inf") for w in SEQUENCE)


def test_inf_norm_is_applied_with_coefficient_zero():
    """One +Inf entry: coefficient 0, so Adadelta's square_avg and acc_delta decay by rho, the parameter does not
    move except at the Inf entry (NaN), and the step counts."""
    p0 = [np.array([1.0, -2.0, 3.0]), np.array([0.5, 0.25])]
    ref = optim_ref.Optimizer(p0, "Adadelta", lr=1.0, eps=1e-6)
    ref.state1 = [np.array([4.0, 1.0, 2.0]), np.array([1.0, 8.0])]
    ref.state2 = [np.array([1e-4, 2e-4, 3e-4]), np.array([5e-4, 6e-4])]
    s1, s2 = [s.copy() for s in ref.state1], [s.copy() for s in ref.state2]
    norm, did = ref.step([np.array([1.0, np.inf, -1.0]), np.array([2.0, 3.0])])
    assert math.isinf(norm) and did and ref.n_steps == 1 and optim_ref.clip_coef(norm) == 0.0
    assert np.array_equal(np.isnan(ref.params[0]), [False, True, False])
    assert np.array_equal(ref.params[0][[0, 2]], p0[0][[0, 2]]) and np.array_equal(ref.params[1], p0[1])
    np.testing.assert_allclose(ref.state1[1], 0.9 * s1[1], rtol=1e-15)
    np.testing.assert_allclose(ref.state2[0][[0, 2]], 0.9 * s2[0][[0, 2]], rtol=1e-15)

