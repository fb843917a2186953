"""Encoder / attention building blocks with the reference's constructor signatures and state_dict keys
(/root/reference/src/module.py), computing through the b200asr kernels.

  RNNLayer               -> persistent BiLSTM kernels (ops.bilstm) + cuBLAS input/weight-grad GEMMs
  LocationAwareAttention -> fused single-launch attention step (ops.loc_attention_step)
  CNNExtractor / VGGExtractor / ScaleDotAttention -> library convolutions / GEMMs (cuDNN, cuBLAS); these are
      plain dense contractions outside the four north-star kernels (SURVEY.md 8(f) rank 4).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops


class VGGExtractor(nn.Module):
    """VGG-like prenet (src/module.py:7-66): 2x(conv3x3-ReLU x2 + maxpool 2x2); time and frequency /4."""

    def __init__(self, input_dim):
        super().__init__()
        self.init_dim = 64
        self.hide_dim = 128
        in_channel, freq_dim, out_dim = self.check_dim(input_dim)
        self.in_channel, self.freq_dim, self.out_dim = in_channel, freq_dim, out_dim
        c0, c1 = self.init_dim, self.hide_dim
        self.extractor = nn.Sequential(
            nn.Conv2d(in_channel, c0, 3, stride=1, padding=1), nn.ReLU(),
            nn.Conv2d(c0, c0, 3, stride=1, padding=1), nn.ReLU(),
            nn.MaxPool2d(2, stride=2),
            nn.Conv2d(c0, c1, 3, stride=1, padding=1), nn.ReLU(),
            nn.Conv2d(c1, c1, 3, stride=1, padding=1), nn.ReLU(),
            nn.MaxPool2d(2, stride=2))

    def check_dim(self, input_dim):
        if input_dim % 13 == 0:      # MFCC
            return input_dim // 13, 13, (13 // 4) * self.hide_dim
        if input_dim % 40 == 0:      # fbank
            return input_dim // 40, 40, (40 // 4) * self.hide_dim
        raise ValueError("Acoustic feature dimension for VGG should be 13/26/39(MFCC) or 40/80/120(Fbank) but got %d"
                         % input_dim)

    def view_input(self, feature, feat_len):
        feat_len = feat_len // 4
        rem = feature.shape[1] % 4
        if rem != 0:
            feature = feature[:, :-rem, :].contiguous()
        bs, ts, _ = feature.shape
        feature = feature.view(bs, ts, self.in_channel, self.freq_dim).transpose(1, 2)
        return feature, feat_len

    def forward(self, feature, feat_len):
        feature, feat_len = self.view_input(feature, feat_len)
        # Library convolutions, but NOT cuDNN's transform-domain algorithms: on zero-padded frames (exactly 0 activations,
        # zero-initialised biases) Winograd / FFT tiles leave ~1e-9 rounding noise where the exact result is 0, ReLU'(x)
        # then passes gradient where the reference's direct convolution blocks it (measured: the 64->128 / 128->128 bias
        # gradients off by 5-20 %, tools/debug_vgg2.py).  ATen's native direct convolution matches the CPU path.
        with torch.backends.cudnn.flags(enabled=False):
            feature = self.extractor(feature)
        feature = feature.transpose(1, 2)
        feature = feature.contiguous().view(feature.shape[0], feature.shape[1], self.out_dim)
        return feature, feat_len


class CNNExtractor(nn.Module):
    """Two Conv1d(k=4, s=2, p=1) without non-linearity (src/module.py:68-90); time /4."""

    def __init__(self, input_dim, out_dim):
        super().__init__()
        self.out_dim = out_dim
        self.extractor = nn.Sequential(nn.Conv1d(input_dim, out_dim, 4, stride=2, padding=1),
                                       nn.Conv1d(out_dim, out_dim, 4, stride=2, padding=1))

    def forward(self, feature, feat_len):
        feat_len = feat_len // 4
        for conv in self.extractor:             # tensor-core GEMM over the in-place im2col view (ops.Conv1dK4S2Fn)
            feature = ops.conv1d_k4s2p1(feature, conv)
        return feature.contiguous(), feat_len


class RNNLayer(nn.Module):
    """(Bi)LSTM + optional LayerNorm / dropout / time down-sampling / tanh projection (src/module.py:93-158).

    `self.layer` is a torch.nn.LSTM used purely as the parameter container (identical state_dict keys); the
    recurrence itself runs in the persistent sm_90a kernels."""

    def __init__(self, input_dim, module, dim, bidirection, dropout, layer_norm, sample_rate, sample_style, proj):
        super().__init__()
        rnn_out_dim = 2 * dim if bidirection else dim
        self.out_dim = sample_rate * rnn_out_dim if sample_rate > 1 and sample_style == "concat" else rnn_out_dim
        self.dropout = dropout
        self.layer_norm = layer_norm
        self.sample_rate = sample_rate
        self.sample_style = sample_style
        self.proj = proj
        self.ndir = 2 if bidirection else 1
        if self.sample_style not in ["drop", "concat"]:
            raise ValueError("Unsupported Sample Style: " + self.sample_style)
        self.module = module.upper()
        if self.module not in ("LSTM", "GRU"):
            raise NotImplementedError("RNN module %s (the reference accepts LSTM and GRU, src/module.py:112-113)" % module)
        # LSTM: parameter container only, the recurrence runs in the persistent sm_90a kernels.  GRU (SURVEY.md 8(f)
        # rank 4, no BASELINE config uses it): the library cuDNN layer, same state_dict keys as the reference.
        self.layer = getattr(nn, self.module)(input_dim, dim, bidirectional=bidirection, num_layers=1, batch_first=True)
        if self.layer_norm:
            self.ln = nn.LayerNorm(rnn_out_dim)
        if self.dropout > 0:
            self.dp = nn.Dropout(p=dropout)
        if self.proj:
            self.pj = nn.Linear(rnn_out_dim, rnn_out_dim)

    def lstm_params(self):
        ps = []
        for sfx in ["", "_reverse"][:self.ndir]:
            ps += [getattr(self.layer, n + "_l0" + sfx) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        return ps

    def forward(self, input_x, x_len):
        if self.module == "LSTM":
            output = ops.bilstm(input_x, self.lstm_params(), self.ndir)
        else:
            output, _ = self.layer(input_x)
        if self.layer_norm:
            output = self.ln(output)
        if self.dropout > 0:
            output = self.dp(output)
        if self.sample_rate > 1:
            bs, ts, fd = output.shape
            x_len = x_len // self.sample_rate
            if self.sample_style == "drop":
                output = output[:, ::self.sample_rate, :].contiguous()
            else:
                rem = ts % self.sample_rate
                if rem != 0:
                    output = output[:, :-rem, :]
                output = output.contiguous().view(bs, ts // self.sample_rate, fd * self.sample_rate)
        if self.proj:
            output = torch.tanh(ops.linear3x(output, self.pj))
        return output, x_len


class BaseAttention(nn.Module):
    """Masking + softmax + context (src/module.py:161-195)."""

    def __init__(self, temperature, num_head):
        super().__init__()
        self.temperature = temperature
        self.num_head = num_head
        self.softmax = nn.Softmax(dim=-1)
        self.reset_mem()

    def reset_mem(self):
        self.mask = None
        self.k_len = None

    def set_mem(self, prev_att):
        pass

    def compute_mask(self, k, k_len):
        self.k_len = k_len
        bs, ts, _ = k.shape
        pad = torch.arange(ts, device=k.device).unsqueeze(0) >= k_len.to(k.device).unsqueeze(1)   # [B,T] True=pad
        self.mask = pad.unsqueeze(1).expand(bs, self.num_head, ts).reshape(-1, ts)

    def _attend(self, energy, value):
        attn = energy / self.temperature
        attn = attn.masked_fill(self.mask, float("-inf"))
        attn = self.softmax(attn)
        output = torch.bmm(attn.unsqueeze(1), value).squeeze(1)
        return output, attn


class ScaleDotAttention(BaseAttention):
    """Scaled dot-product attention (src/module.py:198-212); library bmm path."""

    def forward(self, q, k, v):
        ts = k.shape[1]
        energy = torch.bmm(q.unsqueeze(1), k.transpose(1, 2)).squeeze(1)
        output, attn = self._attend(energy, v)
        return output, attn.view(-1, self.num_head, ts)


class LocationAwareAttention(BaseAttention):
    """Location-aware attention (src/module.py:215-258).  With one head (every BASELINE config) the whole step -
    conv over the previous alignment, location projection, energy, masked softmax, context - is ONE kernel launch
    (ops.loc_attention_step); multi-head falls back to the unfused library ops."""

    def __init__(self, kernel_size, kernel_num, dim, num_head, temperature):
        super().__init__(temperature, num_head)
        self.prev_att = None
        self.loc_conv = nn.Conv1d(num_head, kernel_num, kernel_size=2 * kernel_size + 1, padding=kernel_size,
                                  bias=False)
        self.loc_proj = nn.Linear(kernel_num, dim, bias=False)
        self.gen_energy = nn.Linear(dim, 1)
        self.dim = dim
        self._mem = None

    def reset_mem(self):
        super().reset_mem()
        self.prev_att = None
        self._mem = None

    def set_mem(self, prev_att):
        self.prev_att = prev_att

    def init_prev_att(self, bs, ts, device):
        lens = self.k_len.to(device=device, dtype=torch.float32).clamp_min(1.0)
        valid = torch.arange(ts, device=device).unsqueeze(0) < self.k_len.to(device).unsqueeze(1)
        att = valid.to(torch.float32) / lens.unsqueeze(1)
        return att.unsqueeze(1).expand(bs, self.num_head, ts).contiguous()

    def forward(self, q, k, v):
        bs_nh, ts, _ = k.shape
        bs = bs_nh // self.num_head
        if self.prev_att is None:
            self.prev_att = self.init_prev_att(bs, ts, k.device)
        if self.num_head == 1 and hasattr(ops, "loc_attention_step") and k.is_cuda:
            if getattr(self, "_mem", None) is None:
                # first step of a batch: ONE gradient-accumulator node for key / value / the location weights
                self._mem = ops.attention_memory(k, v, self.loc_conv.weight, self.loc_proj.weight,
                                                 self.gen_energy.weight, self.gen_energy.bias)
            mem, mk, mv, cw, pw, ew, eb, token = self._mem
            output, attn = ops.loc_attention_mem_step(mem, token, q, mk, mv, self.prev_att.view(bs, ts), self.k_len,
                                                      cw, pw, ew, eb, self.temperature)
            attn = attn.view(bs, 1, ts)
        else:
            loc = torch.tanh(self.loc_proj(self.loc_conv(self.prev_att).transpose(1, 2)))
            loc = loc.unsqueeze(1).repeat(1, self.num_head, 1, 1).view(-1, ts, self.dim)
            energy = self.gen_energy(torch.tanh(k + q.unsqueeze(1) + loc)).squeeze(2)
            output, attn = self._attend(energy, v)
            attn = attn.view(bs, self.num_head, ts)
        self.prev_att = attn
        return output, attn
