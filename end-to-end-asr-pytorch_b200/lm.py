"""RNN language model with the reference's interface (src/lm.py:6-44): RNNLM(vocab_size, emb_tying, emb_dim, module, dim,
n_layers, dropout), same parameter containers, state_dict keys and initialisation order, forward(x, lens, hidden=None).

LSTM (the lm_example configuration) runs on this library's kernels:
  - embedding: ATen row gather forward, ops.EmbeddingFn backward (b200asr_embedding_bwd, in place into the gradient);
  - each layer: ops.bilstm(ndir=1), the persistent recurrence plus 3xTF32 input / weight-gradient GEMMs, over the padded
    frames.  A row's outputs at t < len do not depend on later frames, so the packed result is the padded one with the
    output zeroed at t >= len; (h_n, c_n) are read from the output and the cell-state stash at t = len - 1.  Every
    padded target is ignored by the loss, so the gradient at padded frames is exactly zero and the backward is the
    packed gradient without packing;
  - projection: ops.linear3x on `trans`, or with weight tying ops.tied_linear on emb.weight (no bias).
`hidden=` (the beam search's one-token call, src/decode.py:141-148) runs step by step on the decoder's machinery
(ops.decoder_weights / decoder_step + ops.lstm_cell, which takes c_prev).  GRU runs the reference's library sequence
(pack -> nn.GRU -> pad)."""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from . import lib as L
from . import ops


class _DetachedState(Function):
    """(h_n, c_n) of the padded-path forward: values only.  The recurrence kernels start from a zero state and have
    no gradient input for the final state, so a non-zero gradient arriving here is an error, not something to drop."""

    @staticmethod
    def forward(ctx, anchor, h, c):
        ctx.set_materialize_grads(False)
        return h.clone(), c.clone()

    @staticmethod
    def backward(ctx, dh, dc):
        for g in (dh, dc):
            if g is not None and bool((g != 0).any()):
                raise L.B200AsrError("RNNLM: a gradient reached the returned hidden state of a forward without "
                                     "hidden=; that path has no gradient through (h_n, c_n)")
        return None, None, None


def _host_lengths(lens, B):
    lens = torch.as_tensor(lens).to("cpu", torch.int64).reshape(-1)
    if lens.numel() != B:
        raise ValueError("RNNLM: %d lengths for a batch of %d" % (lens.numel(), B))
    if int(lens.min()) < 1:
        raise ValueError("RNNLM: every length must be >= 1 (pack_padded_sequence semantics)")
    return lens


class RNNLM(nn.Module):
    """RNN language model (src/lm.py:6-44)."""

    def __init__(self, vocab_size, emb_tying, emb_dim, module, dim, n_layers, dropout):
        super().__init__()
        self.dim = dim
        self.n_layers = n_layers
        self.emb_tying = emb_tying
        if emb_tying:
            assert emb_dim == dim, "Output dim of RNN should be identical to embedding if using weight tying."
        self.vocab_size = vocab_size
        self.emb = nn.Embedding(vocab_size, emb_dim)
        self.dp1 = nn.Dropout(dropout)
        self.dp2 = nn.Dropout(dropout)
        self.module = module.upper()
        if self.module not in ("LSTM", "GRU"):
            raise NotImplementedError("RNNLM module %s (the reference takes nn.LSTM or nn.GRU)" % module)
        self.rnn = getattr(nn, self.module)(emb_dim, dim, num_layers=n_layers, dropout=dropout, batch_first=True)
        if not self.emb_tying:
            self.trans = nn.Linear(dim, vocab_size)
        self.dropout = dropout

    def create_msg(self):
        return ["Model spec.| RNNLM weight tying = {}, # of layers = {}, dim = {}".format(
            self.emb_tying, self.n_layers, self.dim)]

    def _layer_params(self, l):
        return [getattr(self.rnn, "%s_l%d" % (n, l)) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]

    def _project(self, h):
        h = self.dp2(h)
        if self.emb_tying:
            return ops.tied_linear(h, self.emb.weight)
        return ops.linear3x(h, self.trans)

    def forward(self, x, lens, hidden=None):
        """x [B, T] token ids, lens [B] (host or device; >= 1) -> (outputs [B, max(lens), V], hidden).  outputs at
        t >= lens[b] are the projection of a zero state (trans.bias, or 0 when tied), as after pad_packed_sequence."""
        B = x.shape[0]
        lens_h = _host_lengths(lens, B)
        T = int(lens_h.max())
        x = x[:, :T]
        if self.module == "GRU":
            emb_x = self.dp1(self.emb(x))
            if not self.training:
                self.rnn.flatten_parameters()
            packed = nn.utils.rnn.pack_padded_sequence(emb_x, lens_h, batch_first=True, enforce_sorted=False)
            outputs, hidden = self.rnn(packed, hidden)
            outputs, _ = nn.utils.rnn.pad_packed_sequence(outputs, batch_first=True)
            return self._project(outputs), hidden
        if not x.is_cuda:
            raise L.B200AsrError("RNNLM: the LSTM path runs on the CUDA kernels only (got a %s tensor)" % x.device)
        emb_x = self.dp1(ops.embedding(x, self.emb.weight))
        lens_d = lens_h.to(x.device)
        mask = (torch.arange(T, device=x.device).unsqueeze(0) < lens_d.unsqueeze(1)).unsqueeze(-1).to(emb_x.dtype)
        if hidden is None:
            outputs, hidden = self._forward_padded(emb_x, lens_d, mask)
        else:
            outputs, hidden = self._forward_stepwise(emb_x, lens_d, mask, hidden)
        return self._project(outputs), hidden

    def _forward_padded(self, emb_x, lens_d, mask):
        B = emb_x.shape[0]
        rows = torch.arange(B, device=emb_x.device)
        last = lens_d - 1
        h = emb_x
        hn, cn = [], []
        for l in range(self.n_layers):
            sink = ops.CStateSink()
            out = ops.bilstm(h, self._layer_params(l), 1, sink) * mask
            hn.append(out.detach()[rows, last])
            cn.append(sink.cstate[0, rows, last])
            h = out
            if self.dropout > 0 and l + 1 < self.n_layers:
                h = F.dropout(h, self.dropout, self.training)
        return h, _DetachedState.apply(h, torch.stack(hn, 0), torch.stack(cn, 0))

    def _forward_stepwise(self, emb_x, lens_d, mask, hidden):
        B, T, _ = emb_x.shape
        H = self.dim
        h_prev, c_prev = hidden
        if h_prev.shape != (self.n_layers, B, H) or c_prev.shape != (self.n_layers, B, H):
            raise ValueError("RNNLM: hidden must be (h, c) of shape [%d, %d, %d]" % (self.n_layers, B, H))
        hs = [h_prev[l].to(emb_x.device, torch.float32) for l in range(self.n_layers)]
        cs = [c_prev[l].to(emb_x.device, torch.float32) for l in range(self.n_layers)]
        dws = []
        for l in range(self.n_layers):
            I = self.rnn.input_size if l == 0 else H
            if not ops.decoder_gemm_supported(I, H):
                raise L.B200AsrError("RNNLM hidden=: the step GEMM needs (input + hidden) %% 4 == 0 (I=%d H=%d)" % (I, H))
            dws.append(ops.decoder_weights(*self._layer_params(l)))
        outs, h_steps, c_steps = [], [], []
        for t in range(T):
            inp = emb_x[:, t]
            for l in range(self.n_layers):
                pre = ops.decoder_step(dws[l], inp, hs[l])
                hs[l], cs[l] = ops.lstm_cell(pre, cs[l])
                inp = hs[l]
                if self.dropout > 0 and l + 1 < self.n_layers:
                    inp = F.dropout(inp, self.dropout, self.training)
            outs.append(hs[-1])
            h_steps.append(torch.stack(hs, 1))          # [B, n_layers, H]
            c_steps.append(torch.stack(cs, 1))
        outputs = torch.stack(outs, 1) * mask
        rows = torch.arange(B, device=emb_x.device)
        last = lens_d - 1
        h_n = torch.stack(h_steps, 1)[rows, last].transpose(0, 1).contiguous()
        c_n = torch.stack(c_steps, 1)[rows, last].transpose(0, 1).contiguous()
        return outputs, (h_n, c_n)
