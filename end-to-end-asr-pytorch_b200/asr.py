"""ASR model with the reference's API surface (/root/reference/src/asr.py): same constructor arguments, same
forward signature and 5-tuple, same attribute names, same state_dict keys - computing through b200asr kernels.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.distributions.categorical import Categorical

from . import ops
from .module import VGGExtractor, CNNExtractor, RNNLayer, ScaleDotAttention, LocationAwareAttention
from .util import init_weights, init_gate


class ASR(nn.Module):
    """Listener (encoder) + CTC head + attention speller.  Drop-in for src/asr.py:12-155."""

    def __init__(self, input_size, vocab_size, init_adadelta, ctc_weight, encoder, attention, decoder, emb_drop=0.0):
        super().__init__()
        assert 0 <= ctc_weight <= 1
        self.vocab_size = vocab_size
        self.ctc_weight = ctc_weight
        self.enable_ctc = ctc_weight > 0
        self.enable_att = ctc_weight != 1
        self.lm = None
        self.last_ctc_argmax = None

        self.encoder = Encoder(input_size, **encoder)
        if self.enable_ctc:
            self.ctc_layer = nn.Linear(self.encoder.out_dim, vocab_size)
        if self.enable_att:
            self.dec_dim = decoder["dim"]
            self.pre_embed = nn.Embedding(vocab_size, self.dec_dim)
            self.embed_drop = nn.Dropout(emb_drop)
            self.decoder = Decoder(self.encoder.out_dim + self.dec_dim, vocab_size, **decoder)
            query_dim = self.dec_dim * self.decoder.layer
            self.attention = Attention(self.encoder.out_dim, query_dim, **attention)

        if init_adadelta:
            self.apply(init_weights)
            if self.enable_att:
                for l in range(self.decoder.layer):
                    init_gate(getattr(self.decoder.layers, "bias_ih_l{}".format(l)))

    def set_state(self, prev_state, prev_attn):
        self.decoder.set_state(prev_state)
        self.attention.set_mem(prev_attn)

    def create_msg(self):
        msg = ["Model spec.| Encoder's downsampling rate of time axis is {}.".format(self.encoder.sample_rate)]
        if self.encoder.vgg:
            msg.append("           | VGG Extractor w/ time downsampling rate = 4 in encoder enabled.")
        if self.encoder.cnn:
            msg.append("           | CNN Extractor w/ time downsampling rate = 4 in encoder enabled.")
        if self.enable_ctc:
            msg.append("           | CTC training on encoder enabled ( lambda = {}).".format(self.ctc_weight))
        if self.enable_att:
            msg.append("           | {} attention decoder enabled ( lambda = {}).".format(
                self.attention.mode, 1 - self.ctc_weight))
        return msg

    def forward(self, audio_feature, feature_len, decode_step, tf_rate=0.0, teacher=None, emb_decoder=None,
                get_dec_state=False):
        """Same contract as src/asr.py:72-155; returns (ctc_output, encode_len, att_output, att_seq, dec_state)."""
        bs = audio_feature.shape[0]
        ctc_output, att_output, att_seq = None, None, None
        dec_state = [] if get_dec_state else None

        encode_feature, encode_len = self.encoder(audio_feature, feature_len)

        if self.enable_ctc:
            logits = ops.linear3x(encode_feature, self.ctc_layer)
            if getattr(self, "fuse_ctc_head", False) and self.training and logits.is_cuda:
                # train step: the log-softmax is fused into the CTC kernels (ops.CTCHeadOutput: logits + row lse + ids)
                ctc_output = ops.ctc_head(logits)
                self.last_ctc_argmax = ctc_output.ids
            else:
                ctc_output, self.last_ctc_argmax = ops.log_softmax(logits, ctc_head=True)

        if self.enable_att:
            decode_step = int(decode_step)
            self.decoder.init_state(bs)
            self.attention.reset_mem()
            last_char = self.pre_embed(torch.zeros((bs,), dtype=torch.long, device=encode_feature.device))
            att_list, output_seq, state_seq = [], [], []
            if teacher is not None:
                teacher = self.embed_drop(self.pre_embed(teacher))
            # with pure teacher forcing the vocabulary projection does not feed back: hoist it out of the loop
            hoist = (teacher is not None) and (tf_rate == 1) and not get_dec_state

            for t in range(decode_step):
                attn, context = self.attention(self.decoder.get_query(), encode_feature, encode_len)
                decoder_input = torch.cat([last_char, context], dim=-1)
                cur_char, d_state = self.decoder(decoder_input, project=not hoist)
                if teacher is not None:
                    if (tf_rate == 1) or (torch.rand(1).item() <= tf_rate):
                        last_char = teacher[:, t, :]
                    else:
                        with torch.no_grad():
                            if (emb_decoder is not None) and emb_decoder.apply_fuse:
                                _, cur_prob = emb_decoder(d_state, cur_char, return_loss=False)
                            else:
                                cur_prob = cur_char.softmax(dim=-1)
                            sampled_char = Categorical(cur_prob).sample()
                        last_char = self.embed_drop(self.pre_embed(sampled_char))
                else:
                    if (emb_decoder is not None) and emb_decoder.apply_fuse:
                        _, cur_char = emb_decoder(d_state, cur_char, return_loss=False)
                    last_char = self.pre_embed(torch.argmax(cur_char, dim=-1))
                if hoist:
                    state_seq.append(d_state)
                else:
                    output_seq.append(cur_char)
                att_list.append(attn)
                if get_dec_state:
                    dec_state.append(d_state)

            if hoist:
                states = torch.stack(state_seq, dim=1)                      # [B, L, dim]
                att_output = self.decoder.project(states)                   # [B, L, V]
            else:
                att_output = torch.stack(output_seq, dim=1)
            att_seq = torch.stack(att_list, dim=2)                          # [B, N, L, T]
            if get_dec_state:
                dec_state = torch.stack(dec_state, dim=1)

        return ctc_output, encode_len, att_output, att_seq, dec_state


class Decoder(nn.Module):
    """Speller: stacked LSTM or GRU stepped one token at a time + vocabulary projection (src/asr.py:158-221).
    `self.layers` (nn.LSTM / nn.GRU) is the parameter container; each step runs one GEMM + the fused cell kernel.
    The hidden state is (h, c) for an LSTM and h alone for a GRU, each [layer, B, dim], as in the reference."""

    def __init__(self, input_dim, vocab_size, module, dim, layer, dropout):
        super().__init__()
        self.in_dim = input_dim
        self.layer = layer
        self.dim = dim
        self.dropout = dropout
        assert module in ["LSTM", "GRU"], NotImplementedError
        self.module = module
        self.hidden_state = None
        self._dw = None
        self.enable_cell = module == "LSTM"
        self.layers = getattr(nn, module)(input_dim, dim, num_layers=layer, dropout=dropout, batch_first=True)
        self.char_trans = nn.Linear(dim, vocab_size)
        self.final_dropout = nn.Dropout(dropout)

    def init_state(self, bs):
        self._dw = None          # per-batch handles of the own-GEMM step path (ops.decoder_weights)
        device = next(self.parameters()).device
        if self.enable_cell:
            self.hidden_state = (torch.zeros((self.layer, bs, self.dim), device=device),
                                 torch.zeros((self.layer, bs, self.dim), device=device))
        else:
            self.hidden_state = torch.zeros((self.layer, bs, self.dim), device=device)
        return None  # the reference returns CPU copies here (a host sync) that ASR.forward never uses

    def set_state(self, hidden_state):
        device = next(self.parameters()).device
        if self.enable_cell:
            self.hidden_state = (hidden_state[0].to(device), hidden_state[1].to(device))
        else:
            self.hidden_state = hidden_state.to(device)

    def get_state(self):
        if self.enable_cell:
            return (self.hidden_state[0].cpu(), self.hidden_state[1].cpu())
        return self.hidden_state.cpu()

    def get_query(self):
        h = self.hidden_state[0] if self.enable_cell else self.hidden_state
        return h.transpose(0, 1).reshape(-1, self.dim * self.layer)

    def project(self, x):
        return ops.linear3x(self.final_dropout(x), self.char_trans)

    def forward(self, x, project=True):
        h_all, c_all = self.hidden_state if self.enable_cell else (self.hidden_state, None)
        hs, cs = [], []
        inp = x
        own = x.is_cuda and all(ops.decoder_gemm_supported(getattr(self.layers, "weight_ih_l%d" % l).shape[1], self.dim)
                                for l in range(self.layer))
        if own and getattr(self, "_dw", None) is None:
            # first step of a batch: packed [W_ih | W_hh] per layer + ONE weight-gradient accumulator node each
            self._dw = [ops.decoder_weights(*(getattr(self.layers, "%s_l%d" % (n, l))
                                              for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")),
                                            cell=self.module)
                        for l in range(self.layer)]
        for l in range(self.layer):
            w_ih = getattr(self.layers, "weight_ih_l%d" % l)
            w_hh = getattr(self.layers, "weight_hh_l%d" % l)
            b_ih = getattr(self.layers, "bias_ih_l%d" % l)
            b_hh = getattr(self.layers, "bias_hh_l%d" % l)
            if own:
                pre = ops.decoder_step(self._dw[l], inp, h_all[l])
            elif self.enable_cell:
                pre = F.linear(inp, w_ih, b_ih) + F.linear(h_all[l], w_hh, b_hh)
            else:
                pre = ops.gru_preact(F.linear(inp, w_ih, b_ih), F.linear(h_all[l], w_hh, b_hh))
            if self.enable_cell:
                h, c = ops.lstm_cell(pre, c_all[l])
                cs.append(c)
            else:
                h = ops.gru_cell(pre, h_all[l])
            hs.append(h)
            inp = h
            if self.dropout > 0 and l + 1 < self.layer:
                inp = F.dropout(inp, self.dropout, self.training)
        self.hidden_state = (torch.stack(hs, 0), torch.stack(cs, 0)) if self.enable_cell else torch.stack(hs, 0)
        out = inp
        char = self.project(out) if project else None
        return char, out


class Attention(nn.Module):
    """Query/key/value projections + head handling around the attention kernel (src/asr.py:224-313)."""

    def __init__(self, v_dim, q_dim, mode, dim, num_head, temperature, v_proj, loc_kernel_size, loc_kernel_num):
        super().__init__()
        self.v_dim = v_dim
        self.dim = dim
        self.mode = mode.lower()
        self.num_head = num_head
        self.proj_q = nn.Linear(q_dim, dim * num_head)
        self.proj_k = nn.Linear(v_dim, dim * num_head)
        self.v_proj = v_proj
        if v_proj:
            self.proj_v = nn.Linear(v_dim, v_dim * num_head)
        if self.mode == "dot":
            self.att_layer = ScaleDotAttention(temperature, self.num_head)
        elif self.mode == "loc":
            self.att_layer = LocationAwareAttention(loc_kernel_size, loc_kernel_num, dim, num_head, temperature)
        else:
            raise NotImplementedError
        if self.num_head > 1:
            self.merge_head = nn.Linear(v_dim * num_head, v_dim)
        self.key = None
        self.value = None
        self.mask = None

    def reset_mem(self):
        self.key = None
        self.value = None
        self.mask = None
        self.att_layer.reset_mem()

    def set_mem(self, prev_attn):
        self.att_layer.set_mem(prev_attn)

    def forward(self, dec_state, enc_feat, enc_len):
        bs, ts, _ = enc_feat.shape
        query = torch.tanh(self.proj_q(dec_state)).view(bs * self.num_head, self.dim)
        if self.key is None:
            self.att_layer.compute_mask(enc_feat, enc_len.to(enc_feat.device))
            self.key = torch.tanh(ops.linear3x(enc_feat, self.proj_k))
            self.value = torch.tanh(ops.linear3x(enc_feat, self.proj_v)) if self.v_proj else enc_feat
            if self.num_head > 1:
                self.key = self.key.view(bs, ts, self.num_head, self.dim).permute(0, 2, 1, 3)
                self.key = self.key.contiguous().view(bs * self.num_head, ts, self.dim)
                if self.v_proj:
                    self.value = self.value.view(bs, ts, self.num_head, self.v_dim).permute(0, 2, 1, 3)
                    self.value = self.value.contiguous().view(bs * self.num_head, ts, self.v_dim)
                else:
                    self.value = self.value.repeat(self.num_head, 1, 1)
        context, attn = self.att_layer(query, self.key, self.value)
        if self.num_head > 1:
            context = self.merge_head(context.view(bs, self.num_head * self.v_dim))
        return attn, context


class Encoder(nn.Module):
    """Listener: optional VGG/CNN prenet + stacked RNN layers (src/asr.py:316-366)."""

    def __init__(self, input_size, prenet, module, bidirection, dim, dropout, layer_norm, proj, sample_rate,
                 sample_style):
        super().__init__()
        self.vgg = prenet == "vgg"
        self.cnn = prenet == "cnn"
        self.sample_rate = 1
        assert len(sample_rate) == len(dropout), "Number of layer mismatch"
        assert len(dropout) == len(dim), "Number of layer mismatch"
        num_layers = len(dim)
        assert num_layers >= 1, "Encoder should have at least 1 layer"
        module_list = []
        input_dim = input_size
        if self.vgg:
            vgg = VGGExtractor(input_size)
            module_list.append(vgg)
            input_dim = vgg.out_dim
            self.sample_rate *= 4
        if self.cnn:
            cnn = CNNExtractor(input_size, out_dim=dim[0])
            module_list.append(cnn)
            input_dim = cnn.out_dim
            self.sample_rate *= 4
        if module not in ["LSTM", "GRU"]:
            raise NotImplementedError
        for l in range(num_layers):
            module_list.append(RNNLayer(input_dim, module, dim[l], bidirection, dropout[l], layer_norm[l],
                                        sample_rate[l], sample_style, proj[l]))
            input_dim = module_list[-1].out_dim
            self.sample_rate *= sample_rate[l]
        self.in_dim = input_size
        self.out_dim = input_dim
        self.layers = nn.ModuleList(module_list)

    def forward(self, input_x, enc_len):
        for layer in self.layers:
            input_x, enc_len = layer(input_x, enc_len)
        return input_x, enc_len
