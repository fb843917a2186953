"""Static check (no GPU): the VGG path's kernels are in the built library, and the conv-mode instantiations of the
3xTF32 GEMM (conv3x3_gemm_kernel, the gemm3x_kernel body) are wgmma (HGMMA) + TMA (UTMALDG) kernels like the other
forms."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("c++filt") is None, reason="needs cuobjdump + c++filt")
@pytest.mark.skipif(not os.path.exists(SO), reason="library not built (run __graft_entry__.build())")
def test_vgg_kernels_and_conv_mode_gemm_are_shipped():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_mnemonics
    rows = sass_mnemonics.mnemonic_counts(SO)
    for k in ("vgg_im2col_kernel", "vgg_pool_fwd_kernel", "vgg_pool_bwd_kernel", "vgg_feat_grad_kernel"):
        assert any(k in name for name in rows), k
    conv = {k: v for k, v in rows.items() if "conv3x3_gemm_kernel<" in k}
    assert len(conv) == 2, sorted(rows)                  # tn (forward / input gradient) and nt (weight gradient)
    for name, r in conv.items():
        assert r["HGMMA"] >= 12 and r["UTMALDG"] >= 2 and r["SYNCS"] > 0, (name, r)
