"""CPU ORACLE (test infrastructure, NOT a product path) for the GRU speller (decoder.module: GRU).

  * gru_cell / gru_cell_bwd: float64 numpy GRU step on the cell kernel's layout
    pre [B, 4H] = (gi_r + gh_r, gi_z + gh_z, gi_n, gh_n), in ATen's GRUCell expression order.
  * loc_attention_decode / forward_losses / CpuTrainer: oracle/ref_port's reference port with the speller stepped by
    torch._VF.gru (== nn.GRU's forward, src/asr.py:175-177,214-221); everything around the speller is ref_port's.
Pinned against the running reference by tests/golden/model_grudec.npz (oracle/make_golden_grudec.py).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import ref_port
from .make_golden import tiny_model_cfg


def grudec_model_cfg():
    """The golden `grudec` model: make_golden's hybrid model (loc attention) with a 2-layer GRU speller of dim 32."""
    return dict(tiny_model_cfg("hybrid"), decoder=dict(module="GRU", dim=32, layer=2, dropout=0))


# ------------------------------------------------------------------------------------------------ cell
def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def gru_cell(pre, h_prev):
    """-> (h [B, H], gates [B, 4H] = (r, z, n, gh_n))."""
    H = h_prev.shape[1]
    r, z = _sigmoid(pre[:, :H]), _sigmoid(pre[:, H:2 * H])
    ghn = pre[:, 3 * H:]
    n = np.tanh(pre[:, 2 * H:3 * H] + r * ghn)
    return (h_prev - n) * z + n, np.concatenate([r, z, n, ghn], 1)


def gru_cell_bwd(gates, h_prev, dh):
    """-> (dpre [B, 4H], dh_prev_direct [B, H]) of gru_cell; dh_prev_direct = dh . z (the rest flows through pre)."""
    H = h_prev.shape[1]
    r, z, n, ghn = gates[:, :H], gates[:, H:2 * H], gates[:, 2 * H:3 * H], gates[:, 3 * H:]
    dgin = dh * (1 - z) * (1 - n * n)
    dpre = np.concatenate([dgin * ghn * r * (1 - r), dh * (h_prev - n) * z * (1 - z), dgin, dgin * r], 1)
    return dpre, dh * z


# ------------------------------------------------------------------------------------------------ model
def _gru(P, x, hx, num_layers):
    flat = [P["decoder.layers.%s_l%d" % (n, l)] for l in range(num_layers)
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return torch._VF.gru(x, hx, flat, True, num_layers, 0.0, False, False, True)


def loc_attention_decode(P, att_cfg, dec_cfg, enc, enc_len, teacher_ids, steps):
    """ref_port.loc_attention_decode with a GRU speller (hidden state h only).  Computes in enc's dtype, so a float64
    encoder output gives a float64 decode.  Returns (att_output [B,L,V], att_seq [B,1,L,T])."""
    assert att_cfg["mode"] == "loc" and att_cfg["num_head"] == 1 and not att_cfg["v_proj"]
    assert dec_cfg["module"] == "GRU"
    B, T, _ = enc.shape
    nl = dec_cfg["layer"]
    dev = enc.device
    temp = att_cfg["temperature"]
    key = torch.tanh(F.linear(enc, P["attention.proj_k.weight"], P["attention.proj_k.bias"]))
    pad = torch.arange(T, device=dev)[None, :] >= enc_len.to(dev)[:, None]
    prev = (~pad).to(enc.dtype) / enc_len.to(dev).to(enc.dtype)[:, None]
    h = enc.new_zeros(nl, B, dec_cfg["dim"])
    emb = P["pre_embed.weight"]
    last = emb[torch.zeros(B, dtype=torch.long, device=dev)]
    teach = emb[teacher_ids] if teacher_ids is not None else None
    outs, atts = [], []
    r = att_cfg["loc_kernel_size"]
    for t in range(steps):
        q = torch.tanh(F.linear(h.transpose(0, 1).reshape(B, -1), P["attention.proj_q.weight"],
                                P["attention.proj_q.bias"]))
        conv = F.conv1d(prev.unsqueeze(1), P["attention.att_layer.loc_conv.weight"], padding=r)
        loc = torch.tanh(F.linear(conv.transpose(1, 2), P["attention.att_layer.loc_proj.weight"]))
        e = F.linear(torch.tanh(key + q.unsqueeze(1) + loc), P["attention.att_layer.gen_energy.weight"],
                     P["attention.att_layer.gen_energy.bias"]).squeeze(2)
        a = torch.softmax((e / temp).masked_fill(pad, float("-inf")), dim=-1)
        ctx = torch.bmm(a.unsqueeze(1), enc).squeeze(1)
        prev = a
        y, h = _gru(P, torch.cat([last, ctx], dim=-1).unsqueeze(1), h, nl)
        logit = F.linear(y.squeeze(1), P["decoder.char_trans.weight"], P["decoder.char_trans.bias"])
        last = teach[:, t] if teach is not None else emb[logit.argmax(-1)]
        outs.append(logit)
        atts.append(a.unsqueeze(1))
    return torch.stack(outs, 1), torch.stack(atts, 2)


def forward_losses(P, model_cfg, feat, feat_len, txt):
    """ref_port.forward_losses (tf_rate = 1) for a model with a GRU speller."""
    lam = model_cfg["ctc_weight"]
    assert lam < 1, "a CTC-only model has no speller: use ref_port.forward_losses"
    enc, enc_len = ref_port.encoder(P, model_cfg["encoder"], feat, feat_len)
    txt_len = (txt != 0).sum(-1)
    res = {"encode_len": enc_len, "enc": enc}
    total = 0.0
    if lam > 0:
        lp = F.log_softmax(F.linear(enc, P["ctc_layer.weight"], P["ctc_layer.bias"]), dim=-1)
        ctc = F.ctc_loss(lp.transpose(0, 1), txt, enc_len, txt_len, blank=0, reduction="mean", zero_infinity=False)
        res.update(ctc_output=lp, ctc_loss=ctc)
        total = total + ctc * lam
    L = int(txt_len.max())
    att, seq = loc_attention_decode(P, model_cfg["attention"], model_cfg["decoder"], enc, enc_len, txt, L)
    ce = F.cross_entropy(att.reshape(-1, att.shape[-1]), txt[:, :L].reshape(-1), ignore_index=0)
    res.update(att_output=att, att_seq=seq, att_loss=ce)
    res["total_loss"] = total + ce * (1 - lam)
    return res


class CpuTrainer(ref_port.CpuTrainer):
    """ref_port.CpuTrainer (front end, forward, losses, backward, clip, Adadelta) for a model with a GRU speller."""

    def step(self, waves, texts):
        feat, flen, txt, _ = ref_port.collate(waves, self.audio_cfg, texts)
        for v in self.P.values():
            v.grad = None
        res = forward_losses(self.P, self.model_cfg, feat, flen, txt)
        res["total_loss"].backward()
        used = [k for k, v in self.P.items() if v.grad is not None]
        norm, coef = ref_port.grad_norm_clip([self.P[k].grad for k in used])
        if not math.isnan(float(norm)):
            with torch.no_grad():
                for k in used:
                    ref_port.adadelta_update(self.P[k], self.P[k].grad * coef, self.sq[k], self.acc[k], self.lr, 0.9,
                                             self.eps)
        return float(res["total_loss"].detach()), float(norm)
