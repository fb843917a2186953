"""The cluster-size rule of the wgmma backward's exchange, on the CPU: without a device the cluster occupancy query
cannot be asked, so the planner must fall back to CS = 1 for every shape and cap, and the new kernel instances must use
no local memory beyond the CS = 1 instance's."""
import os
import re
import subprocess

import pytest

from oracle import lstm_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_no_device_means_no_clusters(pkg):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device answers the cluster query")
    lib = pkg.load_library()
    for mode in (0, 16, 32):
        lib.b200asr_debug_set_lstm_mode(mode)
        try:
            for B, H, ndir in ((64, 512, 2), (32, 640, 2), (64, 256, 2), (1, 512, 1)):
                assert lib.b200asr_debug_lstm_cluster(B, H, ndir, 1) == 1
                assert lib.b200asr_debug_lstm_cluster(B, H, ndir, 0) == 1
                # the variant query keeps its 9-field layout and answer
                v = lstm_ref.variant(lib, B, H, ndir, True, mode & 3)
                assert v is not None
        finally:
            lib.b200asr_debug_set_lstm_mode(0)
    assert lib.b200asr_debug_lstm_cluster(0, 512, 2, 1) < 0
    assert lib.b200asr_debug_lstm_cluster(64, 512, 3, 1) < 0


def test_cluster_instances_use_no_local_memory():
    """ptxas: every bilstm_bwd_umma_kernel<UB, CS> instance spills at most the 8 bytes of the CS = 1 instance."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "csrc", "lstm_umma.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                          "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src, "-o", os.devnull],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    spills = re.findall(r"Compiling entry function '(\S*bilstm_bwd_umma_kernelILi(\d+)ELi(\d+)E\S*)'.*?\n.*?\n\s*(\d+) "
                        r"bytes stack frame, (\d+) bytes spill stores", out.stderr)
    assert len(spills) == 6, out.stderr[-2000:]
    for _, ub, cs, frame, st in spills:
        assert int(frame) <= 8 and int(st) <= 8, (ub, cs, frame, st)
