"""GRU speller (decoder.module: GRU), CPU side: the float64 cell oracle, the CPU port of the reference on the golden
model, the packing of the step GEMM's weights, and the model's parameter contract."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import gru_ref
from oracle import ref_port


def test_gru_cell_np_matches_torch_grucell():
    """gru_ref.gru_cell forward and backward against float64 nn.GRUCell autograd, the cell inputs rebuilt from
    the GRUCell's own weights (gi = x.W_ih^T + b_ih, gh = h.W_hh^T + b_hh)."""
    torch.manual_seed(3)
    B, I, H = 5, 7, 6
    cell = torch.nn.GRUCell(I, H).double()
    x = torch.randn(B, I, dtype=torch.float64)
    h = torch.randn(B, H, dtype=torch.float64, requires_grad=True)
    out = cell(x, h)
    dh = torch.randn(B, H, dtype=torch.float64)
    out.backward(dh)
    with torch.no_grad():
        gi = x @ cell.weight_ih.t() + cell.bias_ih
        gh = h @ cell.weight_hh.t() + cell.bias_hh
    pre = torch.cat([gi[:, :2 * H] + gh[:, :2 * H], gi[:, 2 * H:], gh[:, 2 * H:]], 1).numpy()
    hn, gates = gru_ref.gru_cell(pre, h.detach().numpy())
    assert np.abs(hn - out.detach().numpy()).max() < 1e-14
    dpre, dh_direct = gru_ref.gru_cell_bwd(gates, h.detach().numpy(), dh.numpy())
    # chain through the two products: dh_prev = dh.z + [d(r,z) | d gh_n] . W_hh;  dW_hh = [d(r,z) | d gh_n]^T . h
    dgh = np.concatenate([dpre[:, :2 * H], dpre[:, 3 * H:]], 1)
    dgi = dpre[:, :3 * H]
    w_hh = cell.weight_hh.detach().numpy()
    assert np.abs(dh_direct + dgh @ w_hh - h.grad.numpy()).max() < 1e-14
    assert np.abs(dgh.T @ h.detach().numpy() - cell.weight_hh.grad.numpy()).max() < 1e-14
    assert np.abs(dgi.T @ x.numpy() - cell.weight_ih.grad.numpy()).max() < 1e-14
    assert np.abs(dgi.sum(0) - cell.bias_ih.grad.numpy()).max() < 1e-14
    assert np.abs(dgh.sum(0) - cell.bias_hh.grad.numpy()).max() < 1e-14


def test_gru_cell_np_saturated_gates_give_zero_not_nan():
    H = 4
    pre = np.array([[100.0] * H + [-100.0] * H + [50.0] * H + [1e3] * H, [-100.0] * H + [100.0] * H + [-50.0] * H +
                    [-1e3] * H])
    h = np.full((2, H), 3.0)
    _, gates = gru_ref.gru_cell(pre, h)
    dpre, dhp = gru_ref.gru_cell_bwd(gates, h, np.ones((2, H)))
    assert np.isfinite(dpre).all() and np.isfinite(dhp).all()


def test_gru_ref_matches_reference_grudec_model():
    """The CPU port (gru_ref: torch._VF.gru speller) on the golden state_dict reproduces the reference's outputs, losses,
    every gradient and the greedy ids of tests/golden/model_grudec.npz."""
    g = load_golden("model_grudec.npz")
    P = {k[3:]: torch.from_numpy(v).clone().requires_grad_(True) for k, v in g.items() if k.startswith("sd.")}
    cfg = gru_ref.grudec_model_cfg()
    feat, flen, txt = (torch.from_numpy(g[k]) for k in ("feat", "feat_len", "txt"))
    res = gru_ref.forward_losses(P, cfg, feat, flen, txt)
    assert np.array_equal(res["encode_len"].numpy(), g["encode_len"])
    assert rel_err(res["ctc_output"].detach().numpy(), g["ctc_output"]) < 1e-5
    assert abs(float(res["ctc_loss"]) - float(g["ctc_loss"])) < 1e-5
    assert rel_err(res["att_output"].detach().numpy(), g["att_output"]) < 1e-5
    assert rel_err(res["att_seq"].detach().numpy(), g["att_seq"]) < 1e-5
    assert np.array_equal(res["att_output"].argmax(-1).numpy(), g["att_argmax"])
    assert abs(float(res["att_loss"]) - float(g["att_loss"])) < 1e-5
    res["total_loss"].backward()
    assert abs(float(res["total_loss"]) - float(g["total_loss"])) < 1e-5
    n = 0
    for k, p in P.items():
        if ("grad." + k) in g:
            assert rel_err(p.grad.numpy(), g["grad." + k], floor=1e-4) < 1e-3, k
            n += 1
    assert n == sum(1 for k in g if k.startswith("grad.")) and "grad.decoder.layers.weight_hh_l1" in g
    norm, _ = ref_port.grad_norm_clip([p.grad for p in P.values() if p.grad is not None])
    assert abs(float(norm) - float(g["grad_norm"])) < 1e-5
    with torch.no_grad():
        enc, enc_len = ref_port.encoder(P, cfg["encoder"], feat, flen)
        out, _ = gru_ref.loc_attention_decode(P, cfg["attention"], cfg["decoder"], enc, enc_len, None,
                                               g["greedy_argmax"].shape[1])
    assert np.array_equal(out.argmax(-1).numpy(), g["greedy_argmax"])
    assert rel_err(out.numpy(), g["greedy_output"]) < 1e-5


def test_gru_weight_packing_is_exact(pkg):
    """pack_decoder_weights('GRU') places every weight and bias sum where the cell kernel's layout needs it (zero
    blocks exactly zero), and unpack_decoder_grads is its adjoint: dW_ih / dW_hh / db_* of the packed product."""
    torch.manual_seed(0)
    I, H, B = 7, 5, 3
    w_ih, w_hh = torch.randn(3 * H, I), torch.randn(3 * H, H)
    b_ih, b_hh = torch.randn(3 * H), torch.randn(3 * H)
    wcat, bias = pkg.ops.pack_decoder_weights("GRU", w_ih, w_hh, b_ih, b_hh)
    assert wcat.shape == (4 * H, I + H) and bias.shape == (4 * H,)
    assert torch.equal(wcat[:2 * H, :I], w_ih[:2 * H]) and torch.equal(wcat[:2 * H, I:], w_hh[:2 * H])
    assert torch.equal(wcat[2 * H:3 * H, :I], w_ih[2 * H:]) and torch.equal(wcat[3 * H:, I:], w_hh[2 * H:])
    assert not wcat[2 * H:3 * H, I:].any() and not wcat[3 * H:, :I].any()
    assert torch.equal(bias, torch.cat([b_ih[:2 * H] + b_hh[:2 * H], b_ih[2 * H:], b_hh[2 * H:]]))
    # the packed product equals the reference's gate sums (up to the fp32 rounding of the packed r / z bias sums)
    x, h = torch.randn(B, I, dtype=torch.float64), torch.randn(B, H, dtype=torch.float64)
    pre = torch.cat([x, h], 1) @ wcat.double().t() + bias.double()
    gi = x @ w_ih.double().t() + b_ih.double()
    gh = h @ w_hh.double().t() + b_hh.double()
    assert torch.allclose(pre, pkg.ops.gru_preact(gi, gh), rtol=0, atol=1e-6)
    # adjoint: <dW, pack(W)> over the packed layout == sum of <dW_part, W_part> over the unpacked parameters
    dW, db = torch.randn(4 * H, I + H), torch.randn(4 * H)
    dw_ih, dw_hh, db_ih, db_hh = pkg.ops.unpack_decoder_grads("GRU", dW, db, I)
    assert dw_ih.shape == w_ih.shape and dw_hh.shape == w_hh.shape and db_ih.shape == db_hh.shape == (3 * H,)
    assert torch.equal(dw_ih, torch.cat([dW[:2 * H, :I], dW[2 * H:3 * H, :I]]))
    assert torch.equal(dw_hh, torch.cat([dW[:2 * H, I:], dW[3 * H:, I:]]))
    assert torch.equal(db_ih, db[:3 * H]) and torch.equal(db_hh, torch.cat([db[:2 * H], db[3 * H:]]))
    # the LSTM packing is the plain concatenation it always was
    wl, bl = pkg.ops.pack_decoder_weights("LSTM", torch.randn(8, I), torch.randn(8, 2), torch.ones(8), torch.ones(8))
    assert wl.shape == (8, I + 2) and torch.equal(bl, torch.full((8,), 2.0))


def test_gru_speller_has_reference_state_dict(pkg):
    """An ASR with decoder.module: GRU has the reference's state_dict keys and shapes (nn.GRU inside), the
    reference's hidden-state API, and init_gate's write of 1 over [3H/4, 3H/2) of bias_ih."""
    cfg = gru_ref.grudec_model_cfg()
    torch.manual_seed(0)
    model = pkg.ASR(8, 12, True, **cfg)
    g = load_golden("model_grudec.npz")
    ref = {k[3:]: v.shape for k, v in g.items() if k.startswith("sd.")}
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == {k: tuple(s) for k, s in ref.items()}
    dec = model.decoder
    assert isinstance(dec.layers, torch.nn.GRU) and not dec.enable_cell
    H = dec.dim
    for l in range(dec.layer):
        b = getattr(dec.layers, "bias_ih_l%d" % l).detach()
        assert torch.equal(b[3 * H // 4:3 * H // 2], torch.ones(3 * H // 4))
        assert not b[:3 * H // 4].any() and not b[3 * H // 2:].any()
    dec.init_state(2)
    assert dec.hidden_state.shape == (dec.layer, 2, H)
    dec.set_state(torch.arange(dec.layer * 2 * H, dtype=torch.float32).view(dec.layer, 2, H))
    q = dec.get_query()
    assert q.shape == (2, H * dec.layer) and torch.equal(q[1, H:], dec.hidden_state[1, 1])
    assert torch.equal(dec.get_state(), dec.hidden_state)
