"""Static check (no GPU) of the built f16x3 GEMM kernel: registers only (no local memory), fp16 wgmma with both
operands from shared memory and no TF32 wgmma, and one full drain per chunk body."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")
pytestmark = [
    pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump"),
    pytest.mark.skipif(not os.path.exists(SO), reason="library not built (run __graft_entry__.build())"),
]


def _kernels(flag):
    text = subprocess.run(["cuobjdump", flag, SO], capture_output=True, text=True, check=True).stdout
    out, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function\s*:?\s*(\S+?):?\s*$", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name is not None:
            out[name].append(line)
    funcs = {k: "\n".join(v) for k, v in out.items() if "gemm_f16x3_kernel" in k}
    assert len(funcs) == 1, sorted(funcs)
    return next(iter(funcs.values()))


def test_f16x3_kernel_uses_no_local_memory():
    m = re.search(r"LOCAL:(\d+)", _kernels("--dump-resource-usage"))
    assert m and int(m.group(1)) == 0


def test_f16x3_kernel_issues_fp16_wgmma_only():
    """SASS names an fp16-input HGMMA without a type suffix (.TF32 / .BF16 / .E4M3 mark the others): 2 K blocks x
    4 k16 steps x 3 products per chunk body, both operands as shared-memory descriptors."""
    body = _kernels("-sass")
    mma = re.findall(r"HGMMA\.(\S+) (R\d+), (\S+), (\S+)", body)
    assert len(mma) == 24, len(mma)
    assert all(shape == "64x128x16.F32" for shape, *_ in mma), {m[0] for m in mma}
    assert all(a.startswith("gdesc") for _, _, a, _ in mma)
    assert "TF32" not in body


def test_f16x3_kernel_drains_once_per_chunk():
    body = _kernels("-sass")
    assert len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0", body)) == 1
    assert len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1", body)) == 1
