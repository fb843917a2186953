"""Generate tests/golden/model_grudec.npz by RUNNING the unmodified reference (CPU): make_golden's model recipe on the
GRU-speller model of oracle/gru_ref.grudec_model_cfg().

    python -m oracle.make_golden_grudec     # from the repo root; needs /root/reference
"""
import torch

from . import gru_ref, make_golden, ref_shim

SPEC = ("grudec", 71, 3, 24, 8, 12, 5)          # kind, seed, B, T, D, V, Lmax (make_golden.golden_model)


def main():
    ref_shim.install()
    torch.set_num_threads(1)
    # golden_model() looks its config up by kind name: give it the GRU-speller model under "grudec" for this run
    base = make_golden.tiny_model_cfg
    make_golden.tiny_model_cfg = lambda kind: gru_ref.grudec_model_cfg() if kind == "grudec" else base(kind)
    try:
        make_golden.golden_model(*SPEC)
    finally:
        make_golden.tiny_model_cfg = base


if __name__ == "__main__":
    main()
