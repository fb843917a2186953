"""Generate the RNN-LM goldens tests/golden/lm.npz and lm_plumbing.npz by RUNNING the unmodified reference (CPU):

    python -m oracle.make_golden_lm [lm] [lm_plumbing]      # from the repo root; needs the reference checkout

Same conventions as oracle/make_golden.py (seeded, tiny, written through golden_io so no file exceeds 1 MB); it
writes only the goldens named on the command line (default: both) and leaves every other file under tests/golden/
untouched.
"""
import os
import sys

import numpy as np
import torch

from . import golden_io, ref_shim
from .make_golden import OUT

LM_VARIANTS = {            # name -> (emb_tying, emb_dim, module, dim); V = 12, 2 layers, dropout 0
    "untied": (False, 16, "LSTM", 32),
    "tied": (True, 32, "LSTM", 32),
    "gru": (False, 16, "GRU", 32),
}
LM_ROWS = [[5, 7, 3, 9, 4, 6, 1], [1], [8, 8, 2, 1], [3, 10, 11, 4, 5, 1]]      # token rows ending in <eos> = 1


def lm_batch():
    """The Solver's view of LM_ROWS (bin/train_lm.py:18-23 + 72-78): txt = [<sos>=0 | data], lens counted on the data
    (incl. <eos>, so one row has length 1), input txt[:, :-1], target txt[:, 1:]."""
    data = torch.zeros(len(LM_ROWS), max(len(r) for r in LM_ROWS), dtype=torch.long)
    for i, r in enumerate(LM_ROWS):
        data[i, :len(r)] = torch.tensor(r)
    txt = torch.cat((torch.zeros((data.shape[0], 1), dtype=torch.long), data), dim=1)
    return txt[:, :-1], torch.sum(data != 0, dim=-1), txt[:, 1:]


def golden_lm():
    """The reference's RNNLM (src/lm.py) at tiny size: outputs incl. padded positions, hidden, loss, gradients and
    norm of one train-mode forward / backward, and one hidden=-driven T = 1 call as BeamDecoder makes it."""
    from src.lm import RNNLM                                                   # the reference's
    V = 12
    x, lens, target = lm_batch()
    out = {"x": x.numpy(), "lens": lens.numpy(), "target": target.numpy()}
    for i, (name, (tying, emb_dim, module, dim)) in enumerate(LM_VARIANTS.items()):
        torch.manual_seed(100 + i)
        model = RNNLM(V, tying, emb_dim, module, dim, 2, 0)
        model.train()
        pred, hidden = model(x, lens)
        loss = torch.nn.CrossEntropyLoss(ignore_index=0)(pred.reshape(-1, V), target.reshape(-1))
        loss.backward()
        p = name + "."
        out[p + "pred"] = pred.detach().numpy()
        out[p + "loss"] = loss.detach().numpy()
        h_n, c_n = hidden if module == "LSTM" else (hidden, None)
        out[p + "h_n"] = h_n.detach().numpy()
        if c_n is not None:
            out[p + "c_n"] = c_n.detach().numpy()
        sq = 0.0
        for k, v in model.named_parameters():
            out[p + "grad." + k] = v.grad.numpy()
            sq += float((v.grad.double() ** 2).sum())
        out[p + "grad_norm"] = np.float64(np.sqrt(sq))
        for k, v in model.state_dict().items():
            out[p + "sd." + k] = v.numpy()
        # BeamDecoder (src/decode.py:141-148): lm(prev_token [B, 1], ones, hidden=prev), eval mode
        model.eval()
        step_x = torch.tensor([[4], [1], [9], [2]])
        prev = tuple(h.detach() for h in hidden) if module == "LSTM" else hidden.detach()
        with torch.no_grad():
            sp, sh = model(step_x, torch.ones(4, dtype=torch.long), hidden=prev)
        out[p + "step_x"] = step_x.numpy()
        out[p + "step_pred"] = sp.numpy()
        sh_h, sh_c = sh if module == "LSTM" else (sh, None)
        out[p + "step_h"] = sh_h.numpy()
        if sh_c is not None:
            out[p + "step_c"] = sh_c.numpy()
        print("lm.npz", name, "loss", float(loss), "grad_norm", float(np.sqrt(sq)))
    golden_io.save(os.path.join(OUT, "lm.npz"), out)


LM_TRAIN_SENTS = ["A TALE OF TWO CITIES", "IT WAS THE BEST OF TIMES", "IT WAS THE WORST OF TIMES", "WISDOM",
                  "FOOLISHNESS AND BELIEF", "THE SEASON OF LIGHT AND OF DARKNESS",
                  "IT WAS THE SPRING OF HOPE IT WAS THE WINTER OF DESPAIR WE HAD EVERYTHING BEFORE US WE HAD NOTHING "
                  "BEFORE US WE WERE ALL GOING DIRECT TO HEAVEN WE WERE ALL GOING DIRECT THE OTHER WAY IN SHORT",
                  "THE PERIOD WAS SO FAR LIKE THE PRESENT PERIOD"]
LM_DEV_SENTS = ["THERE WERE A KING WITH A LARGE JAW", "AND A QUEEN WITH A PLAIN FACE", "ON THE THRONE OF ENGLAND"]


def lm_text_tree(root):
    """Text-only LibriSpeech-shaped tree for the LM Solver: per split one chapter with a transcript file and an EMPTY
    .flac per utterance (LibriTextDataset only lists the audio files to find their transcripts).  Every sentence has
    a different length, so the length sort does not depend on the file listing order; the longest train sentence
    exceeds HALF_BATCHSIZE_TEXT_LEN characters."""
    for split, spk, sents in (("train-clean-100", "1089", LM_TRAIN_SENTS), ("dev-clean", "2277", LM_DEV_SENTS)):
        d = os.path.join(root, "LibriSpeech", split, spk, "134686")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "%s-134686.trans.txt" % spk), "w") as f:
            for i, text in enumerate(sents):
                name = "%s-134686-%04d" % (spk, i)
                f.write("%s %s\n" % (name, text))
                open(os.path.join(d, name + ".flac"), "wb").close()
    return os.path.join(root, "LibriSpeech")


def lm_plumbing_config(cfg, path, vocab_file):
    """The edits lm_example.yaml needs to run on the fixture (the same for the reference and config/b200/lm_libri.yaml)."""
    cfg["data"]["corpus"].update(path=path, train_split=["train-clean-100"], dev_split=["dev-clean"], batch_size=2)
    cfg["data"]["text"] = {"mode": "character", "vocab_file": vocab_file}
    cfg["hparas"].update(max_step=3, valid_step=2)
    cfg["model"].update(emb_dim=32, dim=32, dropout=0)
    return cfg


def golden_lm_plumbing():
    """The reference's own bin/train_lm.Solver (main.py --lm) on the text fixture from seed 0: the token batches of
    one epoch of its train loader and of the steps in order, per-step loss and grad norm, dev perplexities."""
    import argparse
    import tempfile
    import yaml
    from bin.train_lm import Solver
    from src.data import load_textset
    tmp = tempfile.mkdtemp(prefix="b200asr_lm_plumbing_")
    path = lm_text_tree(tmp)
    vocab = os.path.join(OUT, "character.vocab")
    cfg = yaml.load(open(os.path.join(ref_shim.REF_ROOT, "config", "libri", "lm_example.yaml")), Loader=yaml.FullLoader)
    own = yaml.load(open(os.path.join(os.path.dirname(OUT), "..", "config", "b200", "lm_libri.yaml")),
                    Loader=yaml.FullLoader)
    assert own == cfg, "config/b200/lm_libri.yaml drifted from the reference's lm_example.yaml"
    cfg = lm_plumbing_config(cfg, path, vocab)
    out = {}
    torch.manual_seed(0)
    tr, dv, _, _, _ = load_textset(0, False, False, **cfg["data"])
    epoch = [b.numpy() for b in tr]
    out["epoch_n"] = np.int64(len(epoch))
    for i, b in enumerate(epoch):
        out["epoch%d" % i] = b
    for i, b in enumerate(dv):
        out["dev%d" % i] = b.numpy()
    paras = argparse.Namespace(config="lm_example.yaml", name="lm_plumbing", logdir=os.path.join(tmp, "log"),
                               ckpdir=os.path.join(tmp, "ckpt"), outdir=os.path.join(tmp, "out"), load=None, seed=0,
                               cudnn_ctc=False, njobs=0, cpu=True, no_pin=True, test=False, no_msg=True, lm=True,
                               amp=False, reserve_gpu=0, jit=False, gpu=False, pin_memory=False, verbose=False)
    np.random.seed(0)
    solver = Solver(cfg, paras, "train")
    solver.load_data()
    torch.manual_seed(0)                     # weights and loader order are a function of this seed alone
    solver.set_model()
    losses, norms, steps, ppx = [], [], [], []
    real_backward, real_fetch, real_log = solver.backward, solver.fetch_data, solver.write_log

    def backward(loss):
        losses.append(float(loss))
        n = real_backward(loss)
        norms.append(float(n))
        return n

    def fetch(data):
        txt, txt_len = real_fetch(data)
        if solver.model.training:
            steps.append((txt.numpy(), txt_len.numpy()))
        return txt, txt_len

    def write_log(name, d):
        if name == "perplexity" and "dv" in d:
            ppx.append(float(d["dv"]))
        return real_log(name, d)

    solver.backward, solver.fetch_data, solver.write_log = backward, fetch, write_log
    solver.exec()
    for i, (t, l) in enumerate(steps):
        out["step%d_txt" % i] = t
        out["step%d_len" % i] = l
    ck = torch.load(os.path.join(solver.ckpdir, "best_ppx.pth"), map_location="cpu")
    out.update(loss=np.asarray(losses, np.float64), grad_norm=np.asarray(norms, np.float64),
               dev_ppx=np.asarray(ppx, np.float64), best_step=np.int64(ck["global_step"]),
               best_ppx=np.float64(ck["perplexity"]), ckpt_keys=np.asarray(sorted(ck.keys())),
               vocab_size=np.int64(solver.vocab_size))
    for k, v in solver.model.state_dict().items():
        out["final." + k] = v.numpy()
    golden_io.save(os.path.join(OUT, "lm_plumbing.npz"), out)
    print("lm_plumbing.npz loss", losses, "norm", norms, "ppx", ppx)


GOLDENS = {"lm": golden_lm, "lm_plumbing": golden_lm_plumbing}


def main(names=None):
    names = list(names or GOLDENS)
    unknown = [n for n in names if n not in GOLDENS]
    if unknown:
        raise SystemExit("unknown golden(s) %s; choose from %s" % (unknown, sorted(GOLDENS)))
    ref_shim.install()
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(1)
    for n in names:
        GOLDENS[n]()


if __name__ == "__main__":
    main(sys.argv[1:])
