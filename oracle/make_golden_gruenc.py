"""Generate tests/golden/model_gruenc*.npz by RUNNING the unmodified reference (CPU): make_golden's model recipe on a
hybrid model (CTC + location-aware attention) with a 2-layer bidirectional GRU encoder.

    python -m oracle.make_golden_gruenc     # from the repo root; needs /root/reference
"""
import torch

from . import make_golden, ref_shim

# kind, seed, B, T, D, V, Lmax (make_golden.golden_model)
SPEC = ("gruenc", 101, 3, 24, 8, 12, 5)


def gruenc_model_cfg():
    """Layer 0: GRU 8 -> 256 per direction, the width at which the recurrence runs on the wgmma step kernels in both
    passes (b200asr_debug_lstm_variant at B = 3), then a concat pyramid of rate 2 (T / 2, width 1024).  Layer 1: GRU
    1024 -> 16 per direction (the FMA step kernels) with the tanh projection."""
    base = make_golden.tiny_model_cfg("hybrid")
    enc = dict(base["encoder"], module="GRU", dim=[256, 16], sample_rate=[2, 1], sample_style="concat",
               proj=[False, True])
    return dict(base, encoder=enc)


def main():
    ref_shim.install()
    torch.set_num_threads(1)
    base = make_golden.tiny_model_cfg
    make_golden.tiny_model_cfg = lambda kind: gruenc_model_cfg() if kind == "gruenc" else base(kind)
    try:
        make_golden.golden_model(*SPEC)
    finally:
        make_golden.tiny_model_cfg = base


if __name__ == "__main__":
    main()
