"""CPU ORACLE (test infrastructure, NOT a product path) for the RNN language model: a functional restatement of the
reference's LM train step (src/lm.py:31-44, bin/train_lm.py:72-78, torch.optim.Adam) over a `{state_dict key: tensor}`
dictionary, calling the same ATen kernels (nn.LSTM over the packed batch, F.cross_entropy).  It runs on whatever
device and dtype the parameters live on, so the tests use it in fp32 and fp64 at full size.  Clip: ref_port.grad_norm_clip.
"""
import math

import torch
import torch.nn.functional as F


def lm_forward_loss(P, n_layers, x, lens, target, tied=False):
    """Embedding, nn.LSTM over the packed batch, pad, projection, CE(ignore_index=0), dropout 0.
    -> (loss, pred [B, max(lens), V])."""
    emb = P["emb.weight"]
    E, H = emb.shape[1], P["rnn.weight_hh_l0"].shape[1]
    lstm = torch.nn.LSTM(E, H, num_layers=n_layers, batch_first=True).to(device=emb.device, dtype=emb.dtype)
    params = {k[len("rnn."):]: v for k, v in P.items() if k.startswith("rnn.")}
    packed = torch.nn.utils.rnn.pack_padded_sequence(F.embedding(x, emb), lens.cpu(), batch_first=True,
                                                     enforce_sorted=False)
    out, _ = torch.func.functional_call(lstm, params, (packed,))
    out, _ = torch.nn.utils.rnn.pad_packed_sequence(out, batch_first=True)
    pred = F.linear(out, emb) if tied else F.linear(out, P["trans.weight"], P["trans.bias"])
    V = pred.shape[-1]
    return F.cross_entropy(pred.reshape(-1, V), target[:, :pred.shape[1]].reshape(-1), ignore_index=0), pred


def adam_update(p, g, m, v, step, lr, betas=(0.9, 0.999), eps=1e-8):
    """torch.optim.Adam (no weight decay, no amsgrad) for one parameter, in place, in torch's order of operations."""
    m.mul_(betas[0]).add_(g, alpha=1 - betas[0])
    v.mul_(betas[1]).addcmul_(g, g, value=1 - betas[1])
    bc1, bc2 = 1 - betas[0] ** step, 1 - betas[1] ** step
    p.addcdiv_(m, (v.sqrt() / math.sqrt(bc2)).add_(eps), value=-lr / bc1)
