"""Generate tests/golden/model_dot1.npz and model_dotrep.npz by RUNNING the unmodified reference (CPU): make_golden's
model recipe on the scaled dot-product attention models of dotattn_model_cfg().

    python -m oracle.make_golden_dotattn     # from the repo root; needs /root/reference
"""
import torch

from . import make_golden, ref_shim

# kind, seed, B, T, D, V, Lmax (make_golden.golden_model)
SPECS = [("dot1", 81, 3, 24, 8, 12, 5),
         ("dotrep", 91, 4, 26, 8, 12, 6)]


def dotattn_model_cfg(kind):
    """dot1: one head, no value projection, LSTM encoder, attention only (ctc_weight 0).
    dotrep: four heads without a value projection, so Attention.forward's value.repeat(4, 1, 1) makes row b*4 + n
    attend to the encoder states of utterance (b*4 + n) mod B; with B >= 3 ragged utterances that is another
    utterance's states, read up to this utterance's length."""
    base = make_golden.tiny_model_cfg("hybrid")
    att = dict(base["attention"], mode="dot")
    if kind == "dot1":
        return dict(base, ctc_weight=0.0, attention=dict(att, num_head=1, v_proj=False))
    if kind == "dotrep":
        return dict(base, ctc_weight=0.3, attention=dict(att, num_head=4, v_proj=False))
    raise KeyError(kind)


def main():
    ref_shim.install()
    torch.set_num_threads(1)
    # golden_model() looks its config up by kind name: give it the dot-attention models for this run
    base = make_golden.tiny_model_cfg
    make_golden.tiny_model_cfg = lambda kind: dotattn_model_cfg(kind) if kind in ("dot1", "dotrep") else base(kind)
    try:
        for spec in SPECS:
            make_golden.golden_model(*spec)
    finally:
        make_golden.tiny_model_cfg = base


if __name__ == "__main__":
    main()
