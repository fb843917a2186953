"""RNN language model, host side: parameter containers and initialisation against the reference's RNNLM, and the text
pipeline (sorting, bucketing, halving, <sos> insertion, host-side lengths, lm-norm handling, id range checks) against
the batches the reference's own train_lm Solver consumed (tests/golden/lm*.npz)."""
import types

import numpy as np
import pytest
import torch
import yaml

from conftest import ROOT, load_golden
from oracle.make_golden_lm import LM_VARIANTS, lm_plumbing_config, lm_text_tree


@pytest.mark.parametrize("variant", list(LM_VARIANTS))
def test_rnnlm_state_dict_and_seeded_weights_match_reference(pkg, variant):
    g = load_golden("lm.npz")
    tying, emb_dim, module, dim = LM_VARIANTS[variant]
    torch.manual_seed(100 + list(LM_VARIANTS).index(variant))
    model = pkg.RNNLM(12, tying, emb_dim, module, dim, 2, 0)
    ref = {k[len(variant) + 4:]: v for k, v in g.items() if k.startswith(variant + ".sd.")}
    sd = model.state_dict()
    assert list(sd.keys()) == list(ref.keys())
    for k, v in sd.items():
        assert tuple(v.shape) == ref[k].shape, k
        assert np.array_equal(v.numpy(), ref[k]), k           # same seed -> bit-identical initial weights
    assert model.create_msg() == ["Model spec.| RNNLM weight tying = {}, # of layers = 2, dim = {}".format(tying, dim)]


def _config(tmp_path):
    cfg = yaml.safe_load(open(ROOT + "/config/b200/lm_libri.yaml"))
    return lm_plumbing_config(cfg, lm_text_tree(str(tmp_path)), ROOT + "/tests/golden/character.vocab")


def test_text_batches_match_reference_loader(pkg, tmp_path):
    g = load_golden("lm_plumbing.npz")
    cfg = _config(tmp_path)
    torch.manual_seed(0)
    tr, dv, V, tok, _ = pkg.data.load_textset(0, False, False, **cfg["data"])
    assert V == int(g["vocab_size"])
    epoch = [b.numpy() for b in tr]
    assert len(epoch) == int(g["epoch_n"])
    for i, b in enumerate(epoch):
        assert np.array_equal(b, g["epoch%d" % i]), i
    assert min(b.shape[0] for b in epoch) == 1                    # the > 150-token bucket was halved
    dev = [b.numpy() for b in dv]
    assert len(dev) == len([k for k in g if k.startswith("dev") and k[3:].isdigit()])
    for i, b in enumerate(dev):
        assert np.array_equal(b, g["dev%d" % i])


def test_solver_step_batches_sos_and_host_lengths(pkg, tmp_path):
    """The reference seeds, builds the model (which draws from the generator) and then iterates its loader; the same
    sequence here gives the same batches, and fetch_data prepends <sos> and counts the lengths on the host."""
    g = load_golden("lm_plumbing.npz")
    cfg = _config(tmp_path)
    tr, _, V, _, _ = pkg.data.load_textset(0, False, False, **cfg["data"])
    torch.manual_seed(0)
    pkg.RNNLM(V, **cfg["model"])
    stub = types.SimpleNamespace(device=torch.device("cpu"))
    n_steps = len(g["loss"])
    for i, data in enumerate(tr):
        if i == n_steps:
            break
        txt, txt_len = pkg.train_lm.Solver.fetch_data(stub, data)
        assert txt_len.device.type == "cpu"
        assert np.array_equal(txt.numpy(), g["step%d_txt" % i])
        assert np.array_equal(txt_len.numpy(), g["step%d_len" % i])
        assert (txt[:, 0] == 0).all()


def test_lm_norm_file_drops_longest_lines_and_encodes_on_the_fly(pkg, tmp_path, monkeypatch):
    lines = ["AB\n", "ABCDEFG\n", "A\n", "ABCDE\n", "ABC\n", "ABCDEFGHIJ\n"]
    (tmp_path / "librispeech-lm-norm.txt").write_text("".join(lines))
    monkeypatch.setattr(pkg.corpus, "REMOVE_TOP_N_TXT", 2)
    tok = pkg.text.load_text_encoder("character", ROOT + "/tests/golden/character.vocab")
    ds = pkg.corpus.LibriTextDataset(str(tmp_path), ["librispeech-lm-norm.txt"], tok, 1)
    assert len(ds) == 4
    assert ds.text[0] == "ABCDE\n"                                # sorted by raw line length, two longest dropped
    assert ds[0] == tok.encode("ABCDE\n") and ds.text[0] == ds[0]  # encoded when first served, then kept
    bucketed = pkg.corpus.LibriTextDataset(str(tmp_path), ["librispeech-lm-norm.txt"], tok, 2)
    assert bucketed[3] == [tok.encode("AB\n"), tok.encode("A\n")]


def test_synthetic_text_corpus_is_deterministic(pkg):
    a = pkg.data.SyntheticTextDataset(50, 40, 4, seed=3, min_len=2, max_len=30)
    b = pkg.data.SyntheticTextDataset(50, 40, 4, seed=3, min_len=2, max_len=30)
    c = pkg.data.SyntheticTextDataset(50, 40, 4, seed=4, min_len=2, max_len=30)
    assert a.text == b.text and a.text != c.text
    lens = [len(t) for t in a.text]
    assert lens == sorted(lens, reverse=True) and min(lens) >= 2 and max(lens) <= 30
    assert all(t[-1] == 1 and all(3 <= i < 50 for i in t[:-1]) for t in a.text)
    assert len(a[0]) == 4 and a[len(a) - 1] == a.text[-4:]


def test_out_of_range_ids_rejected_on_host(pkg):
    ok = pkg.data.collect_text_batch([[3, 30, 1], [4, 1]], "dev", vocab_size=31)
    assert ok.tolist() == [[3, 30, 1], [4, 1, 0]]
    for bad in ([[3, 31, 1]], [[3, -1, 1]]):
        with pytest.raises(ValueError, match="out of range"):
            pkg.data.collect_text_batch(bad, "dev", vocab_size=31)


def test_halving_only_applies_to_train_buckets(pkg):
    long = [5] * 151 + [1]
    bucket = [[long, long, [3, 1], [4, 1]]]
    assert pkg.data.collect_text_batch(bucket, "train").shape[0] == 2
    assert pkg.data.collect_text_batch(bucket, "dev").shape[0] == 4
