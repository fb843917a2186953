"""Training Solver with the reference's interface (/root/reference/bin/train_asr.py:10-217):
Solver(config, paras, mode).load_data() / .set_model() / .exec(), same loss assembly, validation and checkpoints.
Differences that make it GPU-native: waveforms go to the GPU and the fused front end runs there (fetch_data);
CTC / CE / attention / LSTM are the sm_90a kernels; one process per GPU with a single NCCL grad all-reduce."""
import os

import torch

from . import ops
from .asr import ASR
from .data import load_dataset
from .optim import Optimizer
from .solver import BaseSolver
from .util import cal_er, human_format


class Solver(BaseSolver):
    def __init__(self, config, paras, mode):
        super().__init__(config, paras, mode)
        self.best_wer = {"att": 3.0, "ctc": 3.0}
        self.curriculum = self.config["hparas"]["curriculum"]

    def fetch_data(self, data):
        """(names, wave, wave_len, txt) -> (feat, feat_len, txt, txt_len) on the device: H2D of the raw audio, then
        the fused fbank/delta/CMVN kernels (the reference receives CPU features here, bin/train_asr.py:20-28)."""
        _, wave, wave_len, txt = data
        if self.dp.enabled:          # shard the globally sorted + globally padded batch: rows rank::world
            self.global_batch = wave.shape[0]
            self.global_tokens = float((txt != 0).sum())
            wave, wave_len, txt = self.dp.shard(wave, wave_len, txt)
        wave = wave.to(self.device, non_blocking=True)
        txt = txt.to(self.device, non_blocking=True)
        feat, feat_len = self.audio_transform.batch(wave, wave_len, t_max=None)
        txt_len = torch.sum(txt != 0, dim=-1)
        return feat, feat_len, txt, txt_len

    def load_data(self):
        self.tr_set, self.dv_set, self.feat_dim, self.vocab_size, self.tokenizer, msg = load_dataset(
            self.paras.njobs, self.paras.gpu, self.paras.pin_memory, self.curriculum > 0, device=self.device,
            **self.config["data"])
        self.audio_transform = self.tr_set.audio_transform
        self.verbose(msg)

    def set_model(self):
        init_adadelta = self.config["hparas"]["optimizer"] == "Adadelta"
        self.model = ASR(self.feat_dim, self.vocab_size, init_adadelta, **self.config["model"]).to(self.device)
        self.verbose(self.model.create_msg())
        # in model.train() mode ctc_output is only consumed by CTCLoss and arg-max (exec() below): fuse the CTC head
        self.model.fuse_ctc_head = os.environ.get("B200ASR_FUSE_CTC", "1") == "1"
        self.seq_loss = lambda logits, target: ops.cross_entropy(logits, target, ignore_index=0)
        self.ctc_loss = ops.CTCLoss(blank=0, zero_infinity=False)
        self.emb_fuse, self.emb_reg = False, False
        if ("emb" in self.config) and self.config["emb"]["enable"]:
            raise NotImplementedError("the embedding-regularisation plug-in is outside this hot path")
        self.optimizer = Optimizer([{"params": self.model.parameters()}], **self.config["hparas"])
        if self.dp.enabled:
            torch.distributed.broadcast(self.optimizer.buf.flat, 0)
            self.dp.attach(self.optimizer, self.model)
        self.verbose(self.optimizer.create_msg())
        self.load_ckpt()

    def exec(self):
        self.verbose("Total training steps {}.".format(human_format(self.max_step)))
        ctc_loss, att_loss = None, None
        n_epochs = 0
        self.global_batch = self.global_tokens = None
        self.timer.set()
        while self.step < self.max_step:
            # curriculum hand-off (bin/train_asr.py:86-92): after `curriculum` length-sorted epochs, renew the loader
            # with ascending=False so that sampling becomes random
            if self.curriculum > 0 and n_epochs == self.curriculum:
                self.verbose("Curriculum learning ends after {} epochs, starting random sampling.".format(n_epochs))
                self.tr_set, _, _, _, _, _ = load_dataset(
                    self.paras.njobs, self.paras.gpu, self.paras.pin_memory, False, device=self.device,
                    **self.config["data"])
                self.audio_transform = self.tr_set.audio_transform
            for data in self.tr_set:
                tf_rate = self.optimizer.pre_step(self.step)
                total_loss = 0
                feat, feat_len, txt, txt_len = self.fetch_data(data)
                self.timer.cnt("rd")
                max_len = txt.shape[1] if self.dp.enabled else int(txt_len.max())
                ctc_output, encode_len, att_output, att_align, dec_state = self.model(
                    feat, feat_len, max_len, tf_rate=tf_rate, teacher=txt)
                if ctc_output is not None:
                    self.ctc_loss.global_batch = self.global_batch
                    ctc_loss = self.ctc_loss(ctc_output.transpose(0, 1), txt, encode_len, txt_len)
                    total_loss += ctc_loss * self.model.ctc_weight
                if att_output is not None:
                    b, t, _ = att_output.shape
                    if self.dp.enabled:
                        att_loss = ops.cross_entropy(att_output.reshape(b * t, -1), txt[:, :t].reshape(-1), 0,
                                                     "sum") / self.global_tokens
                    else:
                        att_loss = self.seq_loss(att_output.reshape(b * t, -1), txt[:, :t].reshape(-1))
                    total_loss += att_loss * (1 - self.model.ctc_weight)
                self.timer.cnt("fw")
                grad_norm = self.backward(total_loss)
                self.step += 1
                if (self.step == 1) or (self.step % self.PROGRESS_STEP == 0):
                    self.progress("Tr stat | Loss - {:.2f} | Grad. Norm - {:.2f} | {}".format(
                        total_loss.cpu().item(), grad_norm.item(), self.timer.show()))
                    self.write_log("loss", {"tr_ctc": ctc_loss, "tr_att": att_loss})
                    self.write_log("wer", {"tr_att": cal_er(self.tokenizer, att_output, txt),
                                           "tr_ctc": cal_er(self.tokenizer, ctc_output, txt, ctc=True)})
                if (self.step == 1) or (self.step % self.valid_step == 0):
                    self.validate()
                self.timer.set()
                if self.step > self.max_step:
                    break
            n_epochs += 1
        self.log.close()

    def validate(self):
        self.model.eval()
        dev_wer = {"att": [], "ctc": []}
        for i, data in enumerate(self.dv_set):
            self.progress("Valid step - {}/{}".format(i + 1, len(self.dv_set)))
            dp_on, self.dp.enabled = self.dp.enabled, False       # every rank validates the full dev batch
            feat, feat_len, txt, txt_len = self.fetch_data(data)
            self.dp.enabled = dp_on
            with torch.no_grad():
                ctc_output, encode_len, att_output, att_align, _ = self.model(
                    feat, feat_len, int(int(txt_len.max()) * self.DEV_STEP_RATIO))
            dev_wer["att"].append(cal_er(self.tokenizer, att_output, txt))
            dev_wer["ctc"].append(cal_er(self.tokenizer, ctc_output, txt, ctc=True))
            if i == len(self.dv_set) // 2:
                for j in range(min(len(txt), self.DEV_N_EXAMPLE)):
                    if self.step == 1:
                        self.write_log("true_text{}".format(j), self.tokenizer.decode(txt[j].tolist()))
                    if att_output is not None:
                        self.write_log("att_text{}".format(j),
                                       self.tokenizer.decode(att_output[j].argmax(dim=-1).tolist()))
                    if ctc_output is not None:
                        self.write_log("ctc_text{}".format(j), self.tokenizer.decode(
                            ctc_output[j].argmax(dim=-1).tolist(), ignore_repeat=True))
        for task in ["att", "ctc"]:
            vals = [v for v in dev_wer[task] if v == v]
            dev_wer[task] = sum(vals) / len(vals) if vals else float("nan")
            if dev_wer[task] < self.best_wer[task]:
                self.best_wer[task] = dev_wer[task]
                self.save_checkpoint("best_{}.pth".format(task), "wer", dev_wer[task])
            self.write_log("wer", {"dv_" + task: dev_wer[task]})
        self.save_checkpoint("latest.pth", "wer", dev_wer["att"], show_msg=False)
        self.model.train()
