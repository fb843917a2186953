"""GRU speller (decoder.module: GRU) on the GPU: the cell kernels against float64, the golden model through ASR, two
TrainStep steps against the CPU port of the reference, CUDA-graph replay, the train / greedy-test Solver round trip, and
the library-GEMM fallback for widths the step GEMM does not take.

Cell bound (u = 2^-24, the fp32 unit roundoff; per element, fixed here, independent of any run).  With
A = |gi_n| + |gh_n|: expf / tanhf are within 2 ulp = 4u, so r, z carry <= 6u relative error; the argument
a = gi_n + r.gh_n carries <= 8u.A, hence n <= 12u.(1 + A) absolute.  Then
  h' = (h - n).z + n                      <= 22u.(1 + |h| + A)
  dh_prev = dh.z                          <= 7u.|dh|
  d gi_n = dh.(1 - z).(1 - n^2), d gh_n   <= 35u.|dh|.(1 + A)
  d pre_z = dh.(h - n).z.(1 - z)          <= 20u.|dh|.(1 + |h| + A)
  d pre_r = d gi_n.gh_n.r.(1 - r)         <= 64u.|dh|.(1 + |gh_n|).(1 + A)
and every check below uses K = 64 with those scales (the largest term's constant; 2-3x above the others).
"""
import argparse

import numpy as np
import pytest
import torch
import yaml

import test_gpu_model as gm
from conftest import load_golden, rel_err, scaled_err
from oracle import gru_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
K = 64


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _cell_inputs(B, H, seed):
    g = torch.Generator().manual_seed(seed)
    pre = 60 * torch.rand(B, 4 * H, generator=g) - 30                          # saturating gates at +-30
    far = torch.rand(B, 4 * H, generator=g) < 0.1
    pre[far] = torch.where(torch.rand(int(far.sum()), generator=g) < 0.5, -100.0, 100.0)   # and at +-100
    h = 1e3 * (2 * torch.rand(B, H, generator=g) - 1)                          # h_prev up to 1e3
    dh = torch.randn(B, H, generator=g)
    dh[B // 2] = 0                                                             # a zero dh row
    return pre, h, dh


def _run_cell(pkg, pre, h, dh):
    p = pre.to(DEV).requires_grad_(True)
    hp = h.to(DEV).requires_grad_(True)
    out = pkg.ops.gru_cell(p, hp)
    out.backward(dh.to(DEV))
    return out.detach(), p.grad, hp.grad


@pytest.mark.parametrize("B,H", [(3, 31), (64, 512), (64, 1024)])
def test_gru_cell_matches_float64(pkg, B, H):
    pre, h, dh = _cell_inputs(B, H, seed=B * 7 + H)
    nan_row = B - 1
    pre[nan_row, H // 3] = float("nan")
    out, dpre, dhp = _run_cell(pkg, pre, h, dh)
    out2, dpre2, dhp2 = _run_cell(pkg, pre, h, dh)
    for a, b in ((out, out2), (dpre, dpre2), (dhp, dhp2)):                     # run to run: bit identical
        assert torch.equal(_bits(a), _bits(b))
    out, dpre, dhp = out.cpu().double().numpy(), dpre.cpu().double().numpy(), dhp.cpu().double().numpy()
    pre64, h64, dh64 = pre.double().numpy(), h.double().numpy(), dh.double().numpy()
    ref, gates = gru_ref.gru_cell(pre64, h64)
    rdpre, rdhp = gru_ref.gru_cell_bwd(gates, h64, dh64)
    ok = np.arange(B) != nan_row
    # the NaN stays in its row
    assert np.isnan(out[nan_row]).any() and np.isfinite(out[ok]).all()
    assert np.isfinite(dpre[ok]).all() and np.isfinite(dhp[ok]).all()
    A = np.abs(pre64[:, 2 * H:3 * H]) + np.abs(pre64[:, 3 * H:])
    ah, adh, aghn = np.abs(h64), np.abs(dh64), np.abs(pre64[:, 3 * H:])
    checks = [("h", out, ref, 1 + ah + A),
              ("dh_prev", dhp, rdhp, adh),
              ("d pre_r", dpre[:, :H], rdpre[:, :H], adh * (1 + aghn) * (1 + A)),
              ("d pre_z", dpre[:, H:2 * H], rdpre[:, H:2 * H], adh * (1 + ah + A)),
              ("d gi_n", dpre[:, 2 * H:3 * H], rdpre[:, 2 * H:3 * H], adh * (1 + A)),
              ("d gh_n", dpre[:, 3 * H:], rdpre[:, 3 * H:], adh * (1 + A))]
    for name, got, want, scale in checks:
        err = np.abs(got[ok] - want[ok])
        assert (err <= K * U * scale[ok]).all(), (name, float((err / np.maximum(scale[ok], 1e-30)).max() / U))
    # saturated gates: exactly zero gradient (not NaN); the zero dh row: exactly zero everywhere
    sat_z = np.abs(pre64[:, H:2 * H]) >= 100
    assert (dpre[:, H:2 * H][sat_z & ok[:, None]] == 0).all()
    sat_r = np.abs(pre64[:, :H]) >= 100
    assert (dpre[:, :H][sat_r & ok[:, None]] == 0).all()
    assert (dpre[B // 2] == 0).all() and (dhp[B // 2] == 0).all()


def test_gru_cell_bwd_without_dh(pkg):
    """dh = NULL (h' reaches no loss): every gradient is 0, except the NaN row, which stays NaN only there."""
    L = pkg.lib
    lib = L.load()
    B, H = 64, 512
    pre, h, _ = _cell_inputs(B, H, seed=5)
    pre[7, 3] = float("nan")
    pre_d, h_d = pre.to(DEV), h.to(DEV)
    gates = torch.empty_like(pre_d)
    out = torch.empty_like(h_d)
    L.check(lib.b200asr_gru_cell_fwd(L.ptr(pre_d), L.ptr(h_d), L.ptr(gates), L.ptr(out), B, H, L.stream()))
    dpre = torch.full_like(pre_d, 7.0)
    dhp = torch.full_like(h_d, 7.0)
    L.check(lib.b200asr_gru_cell_bwd(L.ptr(gates), L.ptr(h_d), None, L.ptr(dpre), L.ptr(dhp), B, H, L.stream()))
    dpre, dhp = dpre.cpu(), dhp.cpu()
    ok = torch.arange(B) != 7
    assert (dpre[ok] == 0).all() and (dhp[ok] == 0).all()
    with pytest.raises(pkg.B200AsrError):
        L.check(lib.b200asr_gru_cell_bwd(L.ptr(gates), None, None, L.ptr(dpre.to(DEV)), L.ptr(dhp.to(DEV)), B, H,
                                         L.stream()), "gru_cell_bwd")


# --------------------------------------------------------------------------------------------- golden model grudec
def _tiny_config():
    """test_gpu_model's tiny synthetic-corpus experiment with the golden `grudec` model."""
    return dict(gm._tiny_config("hybrid"), model=gru_ref.grudec_model_cfg())


def _golden_model(pkg):
    g = load_golden("model_grudec.npz")
    model = pkg.ASR(g["feat"].shape[-1], g["sd.ctc_layer.weight"].shape[0], True, **gru_ref.grudec_model_cfg())
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    assert set(sd.keys()) == set(model.state_dict().keys())             # the reference's state_dict contract
    for k, v in model.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    model.load_state_dict(sd)
    return g, model.to(DEV)


def test_grudec_train_step_matches_reference(pkg):
    """CTC and attention outputs, att_seq, both losses, every gradient and the grad-norm of the reference's 2-layer GRU
    speller, to the tolerances of test_gpu_model.test_train_step_matches_reference."""
    g, model = _golden_model(pkg)
    model.train()
    feat, flen, txt = (torch.from_numpy(g[k]).to(DEV) for k in ("feat", "feat_len", "txt"))
    txt_len = (txt != 0).sum(-1)
    ctc_out, enc_len, att_out, att_seq, _ = model(feat, flen, int(txt_len.max()), tf_rate=1.0, teacher=txt)
    assert np.array_equal(enc_len.cpu().numpy(), g["encode_len"])
    assert rel_err(ctc_out.detach().cpu().numpy(), g["ctc_output"]) < 1e-4
    assert np.array_equal(ctc_out.argmax(-1).cpu().numpy(), g["ctc_argmax"])
    assert np.array_equal(model.last_ctc_argmax.cpu().numpy(), g["ctc_argmax"])
    ctc = pkg.CTCLoss(blank=0)(ctc_out.transpose(0, 1), txt, enc_len, txt_len)
    assert abs(ctc.item() - float(g["ctc_loss"])) < 1e-4 * abs(float(g["ctc_loss"]))
    assert rel_err(att_out.detach().cpu().numpy(), g["att_output"],
                   floor=max(1e-3, 0.05 * float(np.abs(g["att_output"]).max()))) < 1e-4
    assert rel_err(att_seq.detach().cpu().numpy(), g["att_seq"], floor=1e-4) < 1e-4
    assert np.array_equal(att_out.argmax(-1).cpu().numpy(), g["att_argmax"])
    b, t, _ = att_out.shape
    ce = pkg.ops.cross_entropy(att_out.view(b * t, -1), txt[:, :t].reshape(-1), ignore_index=0)
    assert abs(ce.item() - float(g["att_loss"])) < 1e-4 * abs(float(g["att_loss"]))
    total = ctc * model.ctc_weight + ce * (1 - model.ctc_weight)
    assert abs(total.item() - float(g["total_loss"])) < 1e-4 * abs(float(g["total_loss"]))
    total.backward()
    sq, n = 0.0, 0
    for k, p in model.named_parameters():
        if "grad." + k in g:
            ref = g["grad." + k]
            assert float(np.abs(p.grad.cpu().numpy() - ref).max()) < 2e-4 * max(float(np.abs(ref).max()), 1e-4), k
            sq += float((p.grad.double() ** 2).sum())
            n += 1
    assert n == sum(1 for k in g if k.startswith("grad.")) and n > 0
    assert abs(np.sqrt(sq) - float(g["grad_norm"])) < 1e-4 * float(g["grad_norm"])


def test_grudec_greedy_ids_bit_exact(pkg):
    g, model = _golden_model(pkg)
    model.eval()
    feat, flen = torch.from_numpy(g["feat"]).to(DEV), torch.from_numpy(g["feat_len"]).to(DEV)
    with torch.no_grad():
        _, _, out, _, _ = model(feat, flen, g["greedy_argmax"].shape[1])
    assert np.array_equal(out.argmax(-1).cpu().numpy(), g["greedy_argmax"])
    assert rel_err(out.cpu().numpy(), g["greedy_output"],
                   floor=max(1e-3, 0.05 * float(np.abs(g["greedy_output"]).max()))) < 1e-4


def test_grudec_two_train_steps_match_cpu_reference_path(pkg):
    """Front end + forward + losses + backward + clip + Adadelta, twice, through TrainStep, against the CPU port of the
    reference's --cpu path with a GRU speller (oracle/gru_ref.CpuTrainer) from identical weights."""
    cfg = _tiny_config()
    step = pkg.TrainStep(cfg, 12, device=DEV, seed=3)
    P = {k: v.detach().cpu().clone() for k, v in step.model.state_dict().items()}
    cpu = gru_ref.CpuTrainer(P, cfg["model"], cfg["data"]["audio"])
    g = torch.Generator().manual_seed(9)
    lens = [9000, 7700, 6400]
    waves = [torch.clamp(0.05 * torch.randn(1, n, generator=g), -1, 1) for n in lens]
    texts = [[3, 4, 4, 5, 1], [6, 7, 1], [8, 9, 10, 1]]
    batch = torch.zeros(3, max(lens))
    txt = torch.zeros(3, 5, dtype=torch.long)
    for i in range(3):
        batch[i, :lens[i]] = waves[i][0]
        txt[i, :len(texts[i])] = torch.tensor(texts[i])
    for it in range(2):
        loss = step(batch.to(DEV), torch.tensor(lens), txt.to(DEV))
        ref_loss, ref_norm = cpu.step(waves, texts)
        assert abs(loss.item() - ref_loss) < 1e-4 * abs(ref_loss), (it, loss.item(), ref_loss)
        assert abs(step.last["grad_norm"].item() - ref_norm) < 2e-4 * ref_norm
    for k, v in step.model.state_dict().items():
        ref = cpu.P[k].detach()
        assert float((v.cpu() - ref).abs().max()) < 2e-4 * max(float(ref.abs().max()), 1e-2), k


def test_grudec_cuda_graph_replay_equals_eager_steps(pkg):
    cfg = _tiny_config()
    g = torch.Generator().manual_seed(11)
    wave = torch.clamp(0.05 * torch.randn(3, 9000, generator=g), -1, 1).to(DEV)
    lens = torch.tensor([9000, 9000, 9000], device=DEV)
    txt = torch.tensor([[3, 4, 4, 5, 1], [6, 7, 1, 0, 0], [8, 9, 10, 1, 0]], device=DEV)
    eager = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    graph = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    assert isinstance(graph.model.decoder.layers, torch.nn.GRU)
    for _ in range(3):
        eager(wave, lens, txt, max_len=5)
    assert graph.capture(wave, lens, txt, warmup=3), graph.graph_error
    for it in range(3):
        le = eager(wave * (1.0 - 0.1 * it), lens, txt, max_len=5)
        lg = graph(wave * (1.0 - 0.1 * it), lens, txt)
        assert abs(le.item() - lg.item()) <= 1e-6 * abs(le.item()), (it, le.item(), lg.item())
    for (k, a), (_, b) in zip(eager.model.state_dict().items(), graph.model.state_dict().items()):
        assert float((a - b).abs().max()) <= 1e-6 * max(float(a.abs().max()), 1e-3), k


def test_grudec_solver_round_trip(pkg, tmp_path):
    """train_asr.Solver (two steps, validation, latest.pth in the reference's dict), then the greedy test_asr.Solver
    from that checkpoint writes both CSVs."""
    cfg = _tiny_config()
    paras = argparse.Namespace(config="tiny.yaml", name="t", logdir=str(tmp_path / "log"), ckpdir=str(tmp_path / "ck"),
                               outdir=str(tmp_path / "out"), load=None, seed=0, njobs=0, gpu=True, pin_memory=False,
                               verbose=False, amp=False)
    tr = pkg.train_asr.Solver(cfg, paras, "train")
    tr.load_data()
    tr.set_model()
    tr.exec()
    assert tr.step >= 2
    ck_path = tmp_path / "ck" / "t" / "latest.pth"
    ck = torch.load(str(ck_path), map_location="cpu")
    assert set(ck.keys()) == {"model", "optimizer", "global_step", "wer"}
    assert set(ck["model"].keys()) == set(tr.model.state_dict().keys())
    assert "decoder.layers.weight_hh_l1" in ck["model"] and ck["model"]["decoder.layers.weight_hh_l1"].shape[0] == 96
    src_yaml = tmp_path / "train.yaml"
    src_yaml.write_text(yaml.safe_dump(cfg))
    dec_cfg = {"src": {"ckpt": str(ck_path), "config": str(src_yaml)},
               "data": {"corpus": {"name": "Synthetic", "dev_split": ["syn"], "test_split": ["syn"], "batch_size": 3,
                                   "n_samples": 8000, "vocab_size": 12}},
               "decode": {"beam_size": 1, "min_len_ratio": 0.01, "max_len_ratio": 0.2}}
    te = pkg.test_asr.Solver(dec_cfg, paras, "test")
    te.load_data()
    te.set_model()
    for k, v in te.model.state_dict().items():
        assert torch.equal(v.cpu(), ck["model"][k]), k
    te.exec()
    for split in ("dev", "test"):
        lines = (tmp_path / "out" / ("t_%s_output.csv" % split)).read_text().splitlines()
        assert lines[0] == "idx\thyp\ttruth" and len(lines) == 1 + 2 * 3


# --------------------------------------------------------------------------------------------- library-GEMM fallback
def test_gru_decoder_fallback_matches_float64_gru(pkg):
    """(I + H) % 4 != 0: the step runs as two library products around the same cell kernel.  Six steps of a 2-layer
    speller against float64 nn.GRU stepped with the same weights: outputs, input and weight gradients."""
    from importlib import import_module
    asr = import_module("end-to-end-asr-pytorch_b200.asr")
    I, H, B, T = 13, 10, 5, 6
    assert not pkg.ops.decoder_gemm_supported(I, H)
    torch.manual_seed(2)
    dec = asr.Decoder(I, 7, "GRU", H, 2, 0.0).to(DEV)
    ref = torch.nn.GRU(I, H, num_layers=2, batch_first=True).double()
    with torch.no_grad():
        for (_, p), (_, q) in zip(dec.layers.named_parameters(), ref.named_parameters()):
            q.copy_(p.double())
    xs = torch.randn(T, B, I)
    gy = torch.randn(T, B, H)
    x_d = xs.to(DEV).requires_grad_(True)
    dec.init_state(B)
    tot = 0
    for t in range(T):
        _, y = dec(x_d[t], project=False)
        tot = tot + (y * gy[t].to(DEV)).sum()
    tot.backward()
    x_r = xs.double().requires_grad_(True)
    hx = torch.zeros(2, B, H, dtype=torch.float64)
    tot_r = 0
    for t in range(T):
        y, hx = ref(x_r[t].unsqueeze(1), hx)
        tot_r = tot_r + (y.squeeze(1) * gy[t].double()).sum()
    tot_r.backward()
    assert scaled_err(dec.hidden_state.detach().cpu().numpy(), hx.detach().numpy()) < 1e-5
    assert scaled_err(x_d.grad.cpu().numpy(), x_r.grad.numpy()) < 1e-5
    for (n, p), (_, q) in zip(dec.layers.named_parameters(), ref.named_parameters()):
        assert scaled_err(p.grad.cpu().numpy(), q.grad.numpy()) < 1e-5, n
