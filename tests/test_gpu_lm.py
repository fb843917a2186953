"""RNN language model on the GPU: golden parity with the reference's RNNLM (untied, tied, GRU), the in-place embedding
gradient kernel against a float64 scatter-add, one lm_example-sized step against the functional oracle in fp32 and
fp64, the train_lm Solver against the reference's own Solver, and main.py --lm end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

from conftest import ROOT, load_golden, rel_err, scaled_err
from oracle import ref_port, ref_port_lm
from oracle.make_golden_lm import LM_VARIANTS, lm_batch, lm_plumbing_config, lm_text_tree

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24


def _rel(a, ref):
    """rel_err with the near-zero floor tied to the tensor's scale, as test_gpu_model.py does for raw outputs."""
    return rel_err(a, ref, floor=max(1e-3, 0.05 * float(np.abs(ref).max())))


def _golden_model(pkg, g, variant):
    tying, emb_dim, module, dim = LM_VARIANTS[variant]
    model = pkg.RNNLM(12, tying, emb_dim, module, dim, 2, 0)
    pre = variant + ".sd."
    model.load_state_dict({k[len(pre):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(pre)})
    return model.to(DEV)


@pytest.mark.parametrize("variant", list(LM_VARIANTS))
def test_lm_matches_reference_golden(pkg, variant):
    g = load_golden("lm.npz")
    p = variant + "."
    model = _golden_model(pkg, g, variant)
    model.train()
    x, lens, target = lm_batch()
    pred, hidden = model(x.to(DEV), lens)
    ref = g[p + "pred"]
    assert pred.shape == ref.shape
    assert _rel(pred.detach().cpu().numpy(), ref) < 1e-4
    # padded positions: the projection of a zero state, exactly
    pad = torch.arange(pred.shape[1]).unsqueeze(0) >= lens.unsqueeze(1)
    padded = pred.detach().cpu()[pad]
    expect = torch.zeros(12) if LM_VARIANTS[variant][0] else model.trans.bias.detach().cpu()
    assert torch.equal(padded, expect.expand_as(padded))
    h_n, c_n = hidden if LM_VARIANTS[variant][2] == "LSTM" else (hidden, None)
    assert _rel(h_n.detach().cpu().numpy(), g[p + "h_n"]) < 1e-4
    if c_n is not None:
        assert _rel(c_n.detach().cpu().numpy(), g[p + "c_n"]) < 1e-4
    loss = pkg.ops.cross_entropy(pred.reshape(-1, 12), target.to(DEV).reshape(-1), ignore_index=0)
    assert abs(loss.item() - float(g[p + "loss"])) < 1e-4 * abs(float(g[p + "loss"]))
    loss.backward()
    sq = 0.0
    for k, prm in model.named_parameters():
        r = g[p + "grad." + k]
        assert float(np.abs(prm.grad.cpu().numpy() - r).max()) < 2e-4 * max(float(np.abs(r).max()), 1e-4), k
        sq += float((prm.grad.double() ** 2).sum())
    assert abs(np.sqrt(sq) - float(g[p + "grad_norm"])) < 1e-4 * float(g[p + "grad_norm"])
    # BeamDecoder's call: one token per row, hidden= the state above, eval mode
    model.eval()
    prev = hidden if c_n is None else (h_n.detach(), c_n.detach())
    with torch.no_grad():
        sp, sh = model(torch.from_numpy(g[p + "step_x"]).to(DEV), torch.ones(4, dtype=torch.long), hidden=prev)
    assert _rel(sp.cpu().numpy(), g[p + "step_pred"]) < 1e-4
    sh_h, sh_c = sh if c_n is not None else (sh, None)
    assert _rel(sh_h.cpu().numpy(), g[p + "step_h"]) < 1e-4
    if sh_c is not None:
        assert _rel(sh_c.cpu().numpy(), g[p + "step_c"]) < 1e-4


def test_hidden_given_matches_padded_path_for_longer_sequences(pkg):
    """hidden= zeros runs the step-by-step path; over T > 1 it must agree with the recurrence kernels."""
    g = load_golden("lm.npz")
    model = _golden_model(pkg, g, "untied").eval()
    x, lens, _ = lm_batch()
    with torch.no_grad():
        a, (ha, ca) = model(x.to(DEV), lens)
        z = torch.zeros(2, 4, 32, device=DEV)
        b, (hb, cb) = model(x.to(DEV), lens, hidden=(z, z))
    assert scaled_err(b.cpu().numpy(), a.cpu().numpy()) < 1e-5
    assert scaled_err(hb.cpu().numpy(), ha.cpu().numpy()) < 1e-5
    assert scaled_err(cb.cpu().numpy(), ca.cpu().numpy()) < 1e-5


def test_gradient_into_returned_hidden_is_refused(pkg):
    g = load_golden("lm.npz")
    model = _golden_model(pkg, g, "untied").train()
    x, lens, _ = lm_batch()
    pred, (h, c) = model(x.to(DEV), lens)
    with pytest.raises(RuntimeError, match="hidden"):
        (pred.sum() + h.sum()).backward()


# ---------------------------------------------------------------------------------------------- embedding kernel
def _scatter64(dW, ids, dy):
    V = dW.shape[0]
    out = dW.double().clone()
    ok = (ids >= 0) & (ids < V)
    out.index_add_(0, ids[ok], dy.double()[ok])
    return out


@pytest.mark.parametrize("N,V,E", [(5000, 16000, 1024), (1, 16000, 64), (3000, 60000, 96), (700, 37, 130)])
def test_embedding_bwd_against_float64(pkg, N, V, E):
    """One token ~2000 times (when N allows), tokens that never occur, ids outside [0, V); V = 60000 keeps the
    per-token counters in global memory, E = 130 is not a multiple of the column block."""
    gen = torch.Generator().manual_seed(N + V)
    ids = torch.randint(0, V // 2, (N,), generator=gen)          # upper half of the vocabulary never occurs
    if N >= 4000:
        ids[torch.randperm(N, generator=gen)[:2000]] = 7
    if N > 10:
        ids[3], ids[N // 2], ids[-1] = -1, V, V + 5
    dy = torch.randn(N, E, generator=gen)
    dW0 = torch.randn(V, E, generator=gen)
    dW0[V - 1] = float("nan")                                    # an untouched row holding NaN
    ids_d, dy_d = ids.to(DEV), dy.to(DEV)
    dW = dW0.to(DEV)
    pkg.ops.embedding_bwd_(dW, ids_d, dy_d)
    got = dW.cpu()
    ref = _scatter64(dW0, ids, dy)
    touched = torch.zeros(V, dtype=torch.bool)
    ok = (ids >= 0) & (ids < V)
    touched[ids[ok]] = True
    assert torch.equal(got[~touched].view(torch.int32), dW0[~touched].view(torch.int32))     # bit for bit, NaN too
    n_tok = torch.bincount(ids[ok], minlength=V).double()
    absum = torch.zeros(V, E, dtype=torch.float64).index_add_(0, ids[ok], dy.double()[ok].abs())
    bound = (n_tok.unsqueeze(1) + 1) * EPS * (absum + dW0.double().abs())
    err = (got.double() - ref).abs()
    assert bool((err[touched] <= bound[touched]).all()), float((err - bound)[touched].max())
    dW2 = dW0.to(DEV)
    pkg.ops.embedding_bwd_(dW2, ids_d, dy_d)
    assert torch.equal(dW2.cpu().view(torch.int32), got.view(torch.int32))                  # two runs bit-identical


def test_tied_embedding_gradient_is_projection_plus_gather(pkg):
    g = load_golden("lm.npz")
    model = _golden_model(pkg, g, "tied").train()
    x, lens, target = lm_batch()
    x = x.to(DEV)
    pred, _ = model(x, lens)
    loss = pkg.ops.cross_entropy(pred.reshape(-1, 12), target.to(DEV).reshape(-1), ignore_index=0)
    loss.backward()
    both = model.emb.weight.grad.clone()
    # the two parts separately, on the same kernels: projection alone (gather input detached), gather alone
    model.emb.weight.grad = None
    emb_x = pkg.ops.embedding(x, model.emb.weight)
    h = emb_x.detach().requires_grad_(True)
    B, T = x.shape
    mask = (torch.arange(T, device=DEV).unsqueeze(0) < lens.to(DEV).unsqueeze(1)).unsqueeze(-1).float()
    out = h
    for l in range(2):
        out = pkg.ops.bilstm(out, model._layer_params(l), 1) * mask
    logits = pkg.ops.tied_linear(out, model.emb.weight)
    pkg.ops.cross_entropy(logits.reshape(-1, 12), target.to(DEV).reshape(-1), ignore_index=0).backward()
    proj = model.emb.weight.grad.clone()
    gather = torch.zeros_like(proj)
    pkg.ops.embedding_bwd_(gather, x, h.grad)
    assert float((both - (proj + gather)).abs().max()) <= 4 * EPS * float((proj.abs() + gather.abs()).max())


# ---------------------------------------------------------------------------------------------- full size
def test_lm_example_sized_step_against_oracle(pkg):
    """V = 16000, E = H = 1024, 2 layers, B = 32, ragged lengths up to 60: the step on the kernels against the
    functional oracle (ATen nn.LSTM with packing) in fp32 (TF32 off) and fp64, then one Adam update."""
    torch.manual_seed(0)
    V, E, B = 16000, 1024, 32
    model = pkg.RNNLM(V, False, E, "LSTM", E, 2, 0).to(DEV)
    gen = torch.Generator().manual_seed(1)
    lens = torch.randint(5, 61, (B,), generator=gen)
    lens[0] = 60
    lens[1] = 1
    x = torch.zeros(B, 60, dtype=torch.long)
    target = torch.zeros(B, 60, dtype=torch.long)
    for b in range(B):
        seq = torch.randint(3, V, (int(lens[b]) + 1,), generator=gen)
        seq[0] = 0
        x[b, :lens[b]] = seq[:-1]
        target[b, :lens[b]] = seq[1:]
    opt = pkg.Optimizer(model.parameters(), "Adam", 1e-4, 1e-8, "fixed")
    opt.pre_step(0)
    P0 = {k: v.detach().clone() for k, v in model.state_dict().items()}
    pred, _ = model(x.to(DEV), lens)
    loss = pkg.ops.cross_entropy(pred.reshape(-1, V), target.to(DEV).reshape(-1), ignore_index=0)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    opt.grad_clip = 5.0
    norm = opt.step()
    new = {k: v.detach().clone() for k, v in model.state_dict().items()}
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        for dt in (torch.float64, torch.float32):
            P = {k: v.to(dt).clone().requires_grad_(True) for k, v in P0.items()}
            rl, rp = ref_port_lm.lm_forward_loss(P, 2, x.to(DEV), lens, target.to(DEV))
            rl.backward()
            assert abs(loss.item() - rl.item()) <= 1e-5 * abs(rl.item()), dt
            assert scaled_err(pred.detach().double().cpu().numpy(), rp.detach().double().cpu().numpy()) < 2e-5, dt
            for k in P:
                bound = 1e-4 if k == "emb.weight" else 5e-4
                assert scaled_err(grads[k].double().cpu().numpy(), P[k].grad.double().cpu().numpy()) < bound, (k, dt)
            rn, _ = ref_port.grad_norm_clip([P[k].grad for k in P])
            assert abs(float(norm) - float(rn)) <= 1e-4 * float(rn)
        # the fused clip + Adam update against torch.optim.Adam's formula on the same (kernel) gradients, in fp64
        coef = min(1.0, 5.0 / (float(norm) + 1e-6))
        for k in P0:
            p = P0[k].double().clone()
            m, v = torch.zeros_like(p), torch.zeros_like(p)
            ref_port_lm.adam_update(p, grads[k].double() * coef, m, v, 1, 1e-4)
            assert float((new[k].double() - p).abs().max()) <= 1e-3 * 1e-4 + 4 * EPS * float(p.abs().max()), k
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


# ---------------------------------------------------------------------------------------------- solver, CLI
def _paras(tmp_path, load=None):
    import argparse
    return argparse.Namespace(config="lm_libri.yaml", name="lm_plumbing", logdir=str(tmp_path / "log"),
                              ckpdir=str(tmp_path / "ckpt"), outdir=str(tmp_path / "out"), load=load, seed=0,
                              cudnn_ctc=False, njobs=0, cpu=False, no_pin=True, test=False, no_msg=True, lm=True,
                              amp=False, reserve_gpu=0, jit=False, gpu=True, pin_memory=False, verbose=False)


def test_solver_matches_reference_solver(pkg, tmp_path):
    g = load_golden("lm_plumbing.npz")
    cfg = yaml.safe_load(open(os.path.join(ROOT, "config", "b200", "lm_libri.yaml")))
    cfg = lm_plumbing_config(cfg, lm_text_tree(str(tmp_path)), os.path.join(ROOT, "tests", "golden", "character.vocab"))
    np.random.seed(0)
    solver = pkg.train_lm.Solver(cfg, _paras(tmp_path), "train")
    solver.load_data()
    torch.manual_seed(0)
    solver.set_model()
    losses, norms, steps, ppx = [], [], [], []
    real_backward, real_fetch, real_log = solver.backward, solver.fetch_data, solver.write_log

    def backward(loss):
        losses.append(float(loss))
        n = real_backward(loss)
        norms.append(float(n))
        return n

    def fetch(data):
        txt, txt_len = real_fetch(data)
        if solver.model.training:
            steps.append((txt.cpu().numpy(), txt_len.numpy()))
        return txt, txt_len

    def write_log(name, d):
        if name == "perplexity" and "dv" in d:
            ppx.append(float(d["dv"]))
        return real_log(name, d)

    solver.backward, solver.fetch_data, solver.write_log = backward, fetch, write_log
    solver.exec()
    assert len(steps) == len(g["loss"])
    for i, (t, l) in enumerate(steps):
        assert np.array_equal(t, g["step%d_txt" % i]) and np.array_equal(l, g["step%d_len" % i])
    assert np.all(np.abs(np.array(losses) - g["loss"]) <= 1e-4 * np.abs(g["loss"]))
    assert np.all(np.abs(np.array(norms) - g["grad_norm"]) <= 5e-4 * g["grad_norm"])
    assert np.all(np.abs(np.array(ppx) - g["dev_ppx"]) <= 1e-4 * g["dev_ppx"])
    ck = torch.load(os.path.join(solver.ckpdir, "best_ppx.pth"), map_location="cpu")
    assert sorted(ck.keys()) == list(g["ckpt_keys"])
    assert ck["global_step"] == int(g["best_step"]) and abs(ck["perplexity"] - float(g["best_ppx"])) < 1e-4 * 31
    # --load resumes at the recorded step with the Adam state restored
    resumed = pkg.train_lm.Solver(cfg, _paras(tmp_path, load=os.path.join(solver.ckpdir, "best_ppx.pth")), "train")
    resumed.load_data()
    resumed.set_model()
    assert resumed.step == ck["global_step"]
    st = resumed.optimizer.get_opt_state_dict()
    for i, s in ck["optimizer"]["state"].items():
        assert torch.equal(st["state"][i]["exp_avg"].cpu(), s["exp_avg"].cpu())
        assert torch.equal(st["state"][i]["exp_avg_sq"].cpu(), s["exp_avg_sq"].cpu())
    assert resumed.optimizer.n_steps == int(float(ck["optimizer"]["state"][0]["step"]))


def test_main_lm_cli_runs_synthetic_config(tmp_path):
    cfg = {"data": {"corpus": {"name": "Synthetic", "path": "", "train_split": ["synthetic"], "dev_split": ["synthetic"],
                               "bucketing": True, "batch_size": 8, "vocab_size": 40, "max_len": 20},
                    "text": {"mode": "character", "vocab_file": "unused"}},
           "hparas": {"valid_step": 2, "max_step": 3, "optimizer": "Adam", "lr": 1e-4, "eps": 1e-8,
                      "lr_scheduler": "fixed"},
           "model": {"emb_tying": True, "emb_dim": 32, "module": "LSTM", "dim": 32, "n_layers": 2, "dropout": 0.5}}
    path = tmp_path / "lm_syn.yaml"
    path.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--config", str(path), "--lm", "--njobs", "0",
                        "--ckpdir", str(tmp_path / "ckpt"), "--logdir", str(tmp_path / "log"), "--no-msg"],
                       capture_output=True, text=True, cwd=str(tmp_path), timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert (tmp_path / "ckpt" / "lm_syn_sd0" / "best_ppx.pth").exists()


def test_dropout_eval_equals_dropout_free_model_and_train_is_finite(pkg):
    g = load_golden("lm.npz")
    ref = _golden_model(pkg, g, "untied").eval()
    model = pkg.RNNLM(12, False, 16, "LSTM", 32, 2, 0.5).to(DEV)
    model.load_state_dict(ref.state_dict())
    x, lens, target = lm_batch()
    model.eval()
    with torch.no_grad():
        a, _ = model(x.to(DEV), lens)
        b, _ = ref(x.to(DEV), lens)
    assert torch.equal(a, b)
    model.train()
    pred, _ = model(x.to(DEV), lens)
    loss = pkg.ops.cross_entropy(pred.reshape(-1, 12), target.to(DEV).reshape(-1), ignore_index=0)
    loss.backward()
    assert np.isfinite(loss.item())
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())
