"""Generate tests/golden/model_loc2.npz and model_locrep.npz by RUNNING the unmodified reference (CPU): make_golden's
model recipe on the multi-head location-aware attention models of locheads_model_cfg().

    python -m oracle.make_golden_locheads     # from the repo root; needs /root/reference
"""
import torch

from . import make_golden, ref_shim

# kind, seed, B, T, D, V, Lmax (make_golden.golden_model)
SPECS = [("loc2", 101, 3, 24, 8, 12, 5),
         ("locrep", 111, 4, 26, 8, 12, 6)]


def locheads_model_cfg(kind):
    """loc2: two heads with a value projection, attention only (ctc_weight 0); loc_conv.weight is [K, 2, 2R+1].
    locrep: four heads without a value projection, so Attention.forward's value.repeat(4, 1, 1) makes row b*4 + n
    attend to the encoder states of utterance (b*4 + n) mod B, read up to the length of utterance b; ctc_weight 0.3."""
    base = make_golden.tiny_model_cfg("hybrid")
    att = dict(base["attention"], mode="loc")
    if kind == "loc2":
        return dict(base, ctc_weight=0.0, attention=dict(att, num_head=2, v_proj=True))
    if kind == "locrep":
        return dict(base, ctc_weight=0.3, attention=dict(att, num_head=4, v_proj=False))
    raise KeyError(kind)


def main():
    ref_shim.install()
    torch.set_num_threads(1)
    # golden_model() looks its config up by kind name: give it the multi-head models for this run
    base = make_golden.tiny_model_cfg
    make_golden.tiny_model_cfg = lambda kind: locheads_model_cfg(kind) if kind in ("loc2", "locrep") else base(kind)
    try:
        for spec in SPECS:
            make_golden.golden_model(*spec)
    finally:
        make_golden.tiny_model_cfg = base


if __name__ == "__main__":
    main()
