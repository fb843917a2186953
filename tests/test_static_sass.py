"""Static check (no GPU): the built library really contains the Hopper paths the design claims - wgmma
(HGMMA), TMA tensor / bulk copies (UTMALDG / UBLKCP) and cp.async (LDGSTS) - in the kernels that
are supposed to use them.  Reads the SASS of the in-tree libb200asr.so with cuobjdump (tools/sass_mnemonics.py)."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("c++filt") is None, reason="needs cuobjdump + c++filt")
@pytest.mark.skipif(not os.path.exists(SO), reason="library not built (run __graft_entry__.build())")
def test_shipped_kernels_contain_wgmma_and_tma():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_mnemonics
    rows = sass_mnemonics.mnemonic_counts(SO)

    def pick(prefix):
        hit = {k: v for k, v in rows.items() if prefix in k}
        assert hit, "no kernel named like %r in the library" % prefix
        return hit

    for name, r in pick("gemm3x_kernel<").items():               # 3xTF32 GEMM: 12 MMAs per K block, TMA loads
        assert r["HGMMA"] >= 12 and r["UTMALDG"] >= 2 and r["SYNCS"] > 0, (name, r)
    for name, r in pick("bilstm_fwd_umma_kernel<").items():      # LSTM forward step: wgmma + bulk-copy state exchange
        assert r["HGMMA"] >= 4 and r["UBLKCP"] >= 6 and r["SYNCS"] > 0, (name, r)
    for name, r in pick("bilstm_bwd_umma_kernel<").items():
        assert r["HGMMA"] >= 4 and r["UBLKCP"] > 0, (name, r)
    for name, r in pick("ctc_alpha_beta_warp_kernel<").items():  # emission look-ahead ring
        assert r["LDGSTS"] > 0, (name, r)
    for name, r in pick("bilstm_fwd_mma_kernel").items():        # the mma.sync fallback generation is still there
        assert r["HMMA"] > 0, (name, r)
