"""The wgmma backward's two-level exchange (clusters of CS unit blocks sum their partials in distributed shared memory
before they reach L2) at every cluster size the planner picks, and at CS = 1 through the debug cap.

Every case runs b200asr_bilstm_fwd / _bwd through the C ABI under the per-row float64 bound of
tests/test_gpu_lstm_variants.py (K * max(err_fp32, 16 * 2^-24)); the extra summation level adds one 2^-24 tag term,
far inside it.  The inputs hold a zero dout row (dG must be exactly 0: tagged zeros are flushed at both levels), dout
rows at 2^-60 .. 2^60 and a NaN in one dout row that must stay in its row.  Two runs must be bit-identical, and the
forward outputs must be bit-equal across cluster sizes (the forward does not use clusters).
"""
import pytest
import torch

from test_gpu_lstm_variants import _bits, _inputs, _parity, _run

pytestmark = pytest.mark.gpu

CAP_MODES = {1: 16, 2: 32, 4: 0}          # debug lstm mode word that caps the cluster size at CS
SHAPES = [(64, 512, 2, 300), (33, 512, 2, 17), (64, 512, 1, 2), (5, 512, 2, 1), (32, 640, 2, 17), (64, 640, 2, 5)]


def _cluster(lib, B, H, ndir, mode):
    lib.b200asr_debug_set_lstm_mode(mode)
    try:
        return lib.b200asr_debug_lstm_cluster(B, H, ndir, 1)
    finally:
        lib.b200asr_debug_set_lstm_mode(0)


def _reachable(lib, B, H, ndir):
    """{CS: mode} for every cluster size the planner picks for the shape under some cap."""
    out = {}
    for cs, mode in sorted(CAP_MODES.items()):
        got = _cluster(lib, B, H, ndir, mode)
        assert 1 <= got <= cs, (B, H, ndir, cs, got)
        out.setdefault(got, mode)
    return out


def test_cfg_b_uses_clusters(pkg):
    """At the cfg-B layer shape the planner picks CS > 1 on this device, and never for the forward."""
    lib = pkg.load_library()
    assert _cluster(lib, 64, 512, 2, 0) in (2, 4)
    assert _cluster(lib, 64, 512, 2, 16) == 1
    assert lib.b200asr_debug_lstm_cluster(64, 512, 2, 0) == 1


@pytest.mark.parametrize("B,H,ndir,T", SHAPES, ids=["B%d-H%d-d%d-T%d" % s for s in SHAPES])
def test_every_cluster_size_vs_fp64(pkg, B, H, ndir, T):
    lib = pkg.load_library()
    reach = _reachable(lib, B, H, ndir)
    assert 1 in reach
    fwd = None
    for cs, mode in sorted(reach.items()):
        ratio, err = _parity(pkg, B, H, ndir, mode, T, seed=B + H + T, dout_nan=(min(3, B - 1), T // 2))
        print("CS=%d: worst row error %.3g (%.3g of the bound)" % (cs, err, ratio))
        pre, whh, dout = _inputs(B, T, H, ndir, seed=B + H + T)
        got = _run(pkg, pre, whh, dout, mode)
        if fwd is None:
            fwd = got[:3]
        else:
            for name, a, b in zip(("out", "cstate", "gates"), fwd, got[:3]):
                assert torch.equal(_bits(a), _bits(b)), (name, "forward differs between cluster sizes", cs)
