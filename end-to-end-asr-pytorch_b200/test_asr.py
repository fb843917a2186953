"""Greedy decoding Solver with the reference's interface (/root/reference/bin/test_asr.py:13-134,199-220): SURVEY.md
8(f) rank 1.  `python main.py --config <decode yaml> --test` with `decode.beam_size: 1` runs the accelerated
`ASR.forward` in argmax-feedback mode over the dev and test sets and writes `<outdir>/<name>_{dev,test}_output.csv`
(`idx<TAB>hyp<TAB>truth`).

GPU-native differences: raw audio goes to the GPU and the fused front end runs there (fetch_data); the arg-max token
ids of a whole batch are produced on the device (for CTC-only models by the log-softmax kernel itself,
`ASR.last_ctc_argmax`) and leave it with ONE copy per batch instead of one `.tolist()` sync per utterance
(bin/test_asr.py:113-118).  Beam search (`beam_size > 1`: src/decode.py, src/ctc.py) is CPU/numpy, batch 1, in the
reference and stays there (DESIGN.md 7)."""
import torch

from .asr import ASR
from .data import load_dataset
from .solver import BaseSolver


def format_hyp_rows(tokenizer, results, collapse_repeats=False):
    """[(idx, [token ids], truth ids)] -> ['idx<TAB>hyp<TAB>truth'] exactly like `write_hyp` in greedy mode
    (bin/test_asr.py:199-217): an empty hypothesis is written as one blank.  The reference computes
    `ignore_repeat = not enable_att` there but never passes it on in greedy mode, so CTC-only hypotheses keep their
    repeated symbols; `collapse_repeats=True` (yaml `decode.ctc_collapse`) applies the evidently intended collapse."""
    rows = []
    for name, hyp_seqs, truth in results:
        hyp = tokenizer.decode(hyp_seqs[0], ignore_repeat=True) if collapse_repeats else tokenizer.decode(hyp_seqs[0])
        if len(hyp) == 0:
            hyp = " "
        rows.append("\t".join([name, hyp, tokenizer.decode(truth)]))
    return rows


class Solver(BaseSolver):
    def __init__(self, config, paras, mode):
        super().__init__(config, paras, mode)
        assert self.config["data"]["corpus"]["name"] == self.src_config["data"]["corpus"]["name"]
        self.config["data"]["corpus"]["path"] = self.src_config["data"]["corpus"]["path"]
        self.config["data"]["corpus"]["bucketing"] = False
        # identical to the training config (bin/test_asr.py:24-28)
        self.config["data"]["audio"] = self.src_config["data"]["audio"]
        self.config["data"]["text"] = self.src_config["data"]["text"]
        self.config["hparas"] = self.src_config["hparas"]
        self.config["model"] = self.src_config["model"]
        self.output_file = str(self.ckpdir) + "_{}_{}.csv"
        self.greedy = self.config["decode"]["beam_size"] == 1
        if not self.greedy:
            raise NotImplementedError("beam_size > 1: beam / CTC-prefix search is the reference's CPU path "
                                      "(src/decode.py, src/ctc.py); only greedy decoding runs on the GPU path")
        self.step = 0

    def fetch_data(self, data):
        _, wave, wave_len, txt = data
        wave = wave.to(self.device, non_blocking=True)
        feat, feat_len = self.audio_transform.batch(wave, wave_len, t_max=None)
        return feat, feat_len, txt, torch.sum(txt != 0, dim=-1)

    def load_data(self):
        self.dv_set, self.tt_set, self.feat_dim, self.vocab_size, self.tokenizer, msg = load_dataset(
            self.paras.njobs, self.paras.gpu, self.paras.pin_memory, False, device=self.device, **self.config["data"])
        self.audio_transform = self.dv_set.audio_transform
        self.verbose(msg)

    def set_model(self):
        init_adadelta = self.config["hparas"]["optimizer"] == "Adadelta"
        self.model = ASR(self.feat_dim, self.vocab_size, init_adadelta, **self.config["model"]).to(self.device)
        if ("emb" in self.config) and self.config["emb"]["enable"]:
            raise NotImplementedError("the embedding-regularisation plug-in is outside this hot path")
        self.load_ckpt()                      # weights only, eval mode
        self.model.eval()
        self.decoder = self.model             # the reference deep-copies the model and deletes the original
        self.verbose(self.decoder.create_msg())

    def greedy_decode(self, dv_set):
        results = []
        ratio = self.config["decode"]["max_len_ratio"]
        bs = self.config["data"]["corpus"]["batch_size"]
        for i, data in enumerate(dv_set):
            self.progress("Valid step - {}/{}".format(i + 1, len(dv_set)))
            feat, feat_len, txt, _ = self.fetch_data(data)
            with torch.no_grad():
                ctc_output, encode_len, att_output, _, _ = self.decoder(
                    feat, feat_len, int(float(feat_len.max()) * ratio), emb_decoder=self.emb_decoder)
                # attention-based if the model has a decoder, else CTC (bin/test_asr.py:113-117); ids stay on the
                # device until the batch is complete
                hyp = att_output.argmax(dim=-1) if att_output is not None else self.decoder.last_ctc_argmax
            hyp = hyp.cpu().tolist()
            truth = txt.tolist()
            for j in range(len(truth)):
                results.append((str(j + bs * i), [hyp[j]], truth[j]))
        return results

    def exec(self):
        collapse = bool(self.config["decode"].get("ctc_collapse", False)) and not self.decoder.enable_att
        for s, ds in zip(["dev", "test"], [self.dv_set, self.tt_set]):
            self.cur_output_path = self.output_file.format(s, "output")
            self.verbose("Performing batch-wise greedy decoding on {} set, num of batch = {}.".format(s, len(ds)))
            results = self.greedy_decode(ds)
            self.verbose("Results will be stored at {}".format(self.cur_output_path))
            with open(self.cur_output_path, "w", encoding="UTF-8") as f:
                f.write("idx\thyp\ttruth\n")
                for row in format_hyp_rows(self.tokenizer, results, collapse):
                    f.write(row + "\n")
        self.verbose("All done !")
