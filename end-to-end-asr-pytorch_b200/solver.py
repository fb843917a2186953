"""BaseSolver with the reference's contract (/root/reference/src/solver.py:13-220): device pick, checkpoint
save/load (same dict keys), logging, and `backward()` = loss.backward + [DP all-reduce] + fused norm/clip/update."""
import abc
import math
import os
import sys

import torch
import yaml

from .dist import DataParallel
from .option import default_hparas
from .util import Timer, human_format


class _NullWriter:
    def add_scalars(self, *a, **k): pass
    def add_text(self, *a, **k): pass
    def add_image(self, *a, **k): pass
    def close(self): pass


class BaseSolver:
    def __init__(self, config, paras, mode):
        self.config, self.paras, self.mode = config, paras, mode
        for k, v in default_hparas.items():
            setattr(self, k, v)
        self.dp = DataParallel()
        if self.paras.gpu and torch.cuda.is_available():
            if self.dp.enabled:
                torch.cuda.set_device(self.dp.local_rank)
            self.device = torch.device("cuda", torch.cuda.current_device())
        else:
            # the reference's --cpu path is the BASELINE (oracle/ref_port.py); this package has no CPU kernels
            raise RuntimeError("the GPU solver needs a CUDA device; run the reference itself for --cpu")
        self.amp = getattr(paras, "amp", False)
        if self.amp:
            raise NotImplementedError("--amp (apex) is not part of the fp32-parity hot path")
        self.exp_name = paras.name
        if self.exp_name is None:
            self.exp_name = paras.config.split("/")[-1].replace(".yaml", "")
            if mode == "train":
                self.exp_name += "_sd{}".format(paras.seed)
        self.emb_decoder = None
        if mode == "train":
            os.makedirs(paras.ckpdir, exist_ok=True)
            self.ckpdir = os.path.join(paras.ckpdir, self.exp_name)
            os.makedirs(self.ckpdir, exist_ok=True)
            self.logdir = os.path.join(paras.logdir, self.exp_name)
            self.log = _NullWriter()
            if self.dp.rank == 0:
                try:
                    from torch.utils.tensorboard import SummaryWriter
                    self.log = SummaryWriter(self.logdir, flush_secs=self.TB_FLUSH_FREQ)
                except Exception:
                    pass
            self.timer = Timer()
            self.step = 0
            self.valid_step = config["hparas"]["valid_step"]
            self.max_step = config["hparas"]["max_step"]
            self.verbose("Exp. name : {}".format(self.exp_name))
            self.verbose("Loading data... large corpus may took a while.")
        elif mode == "test":
            # greedy decoding (SURVEY.md 8(f) rank 1); same bookkeeping as src/solver.py:63-73
            os.makedirs(paras.outdir, exist_ok=True)
            self.ckpdir = os.path.join(paras.outdir, self.exp_name)
            with open(config["src"]["config"], "r") as f:
                self.src_config = yaml.load(f, Loader=yaml.FullLoader)
            self.paras.load = config["src"]["ckpt"]
            self.log = _NullWriter()
            self.step = 0
            self.verbose("Evaluating result of tr. config @ {}".format(config["src"]["config"]))
        else:
            raise NotImplementedError("mode '%s' is outside this hot path" % mode)

    def backward(self, loss):
        """loss.backward(); all-reduce (DP); global norm + clip(GRAD_CLIP) + NaN-skip + optimizer update in fused
        kernels with the norm kept ON THE DEVICE (src/solver.py:76-91 syncs the host on every step)."""
        self.timer.set()
        loss.backward()
        self.optimizer.grad_clip = self.GRAD_CLIP
        grad_norm = self.optimizer.step()
        self.timer.cnt("bw")
        return grad_norm

    def load_ckpt(self):
        if self.paras.load:
            ckpt = torch.load(self.paras.load, map_location=self.device)
            self.model.load_state_dict(ckpt["model"])
            metric, score = "None", 0.0
            for k, v in ckpt.items():
                if type(v) is float:
                    metric, score = k, v
            if self.mode == "train":
                self.step = ckpt["global_step"]
                self.optimizer.load_opt_state_dict(ckpt["optimizer"])
                self.verbose("Load ckpt from {}, restarting at step {} (recorded {} = {:.2f} %)".format(
                    self.paras.load, self.step, metric, score))
            else:
                self.model.eval()
                self.verbose("Evaluation target = {} (recorded {} = {:.2f} %)".format(self.paras.load, metric, score))

    def verbose(self, msg):
        if self.paras.verbose and self.dp.rank == 0:
            for m in (msg if type(msg) == list else [msg]):
                print("[INFO]", m.ljust(100))

    def progress(self, msg):
        if self.paras.verbose and self.dp.rank == 0:
            sys.stdout.write("\033[K")
            print("[{}] {}".format(human_format(self.step), msg), end="\r")

    def write_log(self, log_name, log_dict):
        if type(log_dict) is dict:
            log_dict = {k: (v.item() if torch.is_tensor(v) else v) for k, v in log_dict.items() if v is not None}
            log_dict = {k: v for k, v in log_dict.items() if not math.isnan(v)}
        if log_dict is None:
            return
        if len(log_dict) > 0:
            if "align" in log_name or "spec" in log_name:
                img, form = log_dict
                self.log.add_image(log_name, img, global_step=self.step, dataformats=form)
            elif "text" in log_name or "hyp" in log_name:
                self.log.add_text(log_name, log_dict, self.step)
            else:
                self.log.add_scalars(log_name, log_dict, self.step)

    def save_checkpoint(self, f_name, metric, score, show_msg=True):
        if self.dp.rank != 0:
            return
        ckpt_path = os.path.join(self.ckpdir, f_name)
        torch.save({"model": self.model.state_dict(), "optimizer": self.optimizer.get_opt_state_dict(),
                    "global_step": self.step, metric: score}, ckpt_path)
        if show_msg:
            self.verbose("Saved checkpoint (step = {}, {} = {:.2f}) and status @ {}".format(
                human_format(self.step), metric, score, ckpt_path))

    @abc.abstractmethod
    def load_data(self):
        raise NotImplementedError

    @abc.abstractmethod
    def set_model(self):
        raise NotImplementedError

    @abc.abstractmethod
    def exec(self):
        raise NotImplementedError
