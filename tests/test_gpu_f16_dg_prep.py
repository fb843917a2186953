"""The one-read preparation of a BiLSTM layer's gate gradient dG (ops.f16_split_dg, csrc/gemm.cu): its transposed and
row images and their scales bit-identical to the single-image passes (f16_split_t / f16_split) on the same data, the
column sums (bias gradient) against float64 and bit-identical between runs, dX as one contraction over both
directions against float64, and BiLSTMFn forward + backward at the full BASELINE sizes against float64."""
import pytest
import torch

from conftest import scaled_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _dg(ndir, R, C, seed):
    """N(0,1) gate gradients with rows at 2^+-60, an fp32-subnormal row, an all-zero row chunk, an all-zero column
    chunk (where R allows one), one NaN and one Inf."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(ndir, R, C, device=DEV, generator=gen)
    g[0, min(1, R - 1)] *= 2.0 ** 60
    g[-1, min(2, R - 1)] *= 2.0 ** -60
    g[0, min(3, R - 1)] *= 2.0 ** -135
    g[-1, min(4, R - 1), :min(C, 128)] = 0
    if R >= 256:
        g[0, 128:256, C - 1] = 0
    g[0, R // 2, C // 3] = float("nan")
    g[-1, R - 1, C - 1] = float("inf")
    return g


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


SHAPES = [(2, 64 * 1198, 2048),     # cfg B layer 0 (and 1): 599 full row tiles
          (2, 64 * 599, 2048),      # layer 2: ragged last row tile
          (2, 64 * 299, 2048),      # layer 3
          (2, 15, 192),             # B = 3, T = 5; 4H = 192: a column tail inside the second chunk
          (1, 300, 64)]             # one direction, 4H = 64 (H = 16): one half-empty column chunk


@pytest.mark.parametrize("ndir,R,C", SHAPES)
def test_images_match_the_single_image_passes(pkg, ndir, R, C):
    ops = pkg.ops
    g = _dg(ndir, R, C, R + C)
    gts, (rimg, rsinv), gsum = ops.f16_split_dg(g)
    Kp = pkg.load_library().b200asr_f16x3_padded_k(C)
    assert rimg.shape == (2, R, ndir * Kp) and rsinv.shape == (ndir * Kp // 128, R)
    for d in range(ndir):
        timg, tsinv = gts[d]
        ref_t, ref_ts = ops.f16_split_t(g[d], C, R)
        assert _same(timg, ref_t) and _same(tsinv, ref_ts), d
        ref_r, ref_rs = ops.f16_split(g[d], R, C)
        assert _same(rimg[:, :, d * Kp:(d + 1) * Kp], ref_r), d
        assert _same(rsinv[d * Kp // 128:(d + 1) * Kp // 128], ref_rs), d
    # without the row images: the same transposed operands and sums
    gts2, none, gsum2 = ops.f16_split_dg(g, row_images=False)
    assert none is None and _same(gsum2, gsum)
    for d in range(ndir):
        assert _same(gts2[d][0], gts[d][0]) and _same(gts2[d][1], gts[d][1])


@pytest.mark.parametrize("ndir,R,C", SHAPES)
def test_column_sums_vs_fp64_and_bit_identical(pkg, ndir, R, C):
    ops = pkg.ops
    g = _dg(ndir, R, C, 7 * R + C)
    _, _, gsum = ops.f16_split_dg(g)
    _, _, again = ops.f16_split_dg(g)
    assert _same(gsum, again)
    ref = g.double().sum(1)
    assert torch.equal(torch.isfinite(gsum), torch.isfinite(ref))
    fin = torch.isfinite(ref)
    bound = R * 2.0 ** -24 * g.double().abs().sum(1)
    assert torch.all((gsum.double() - ref).abs()[fin] <= bound[fin])


def _sgemm(a, b):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return a @ b
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _err(out, ref):
    return float((out.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("ndir,R,C,N", [(2, 64 * 1198, 2048, 1024),    # cfg B layer 1: dX over both directions
                                        (2, 64 * 299, 2048, 2048),
                                        (1, 300, 64, 36), (2, 15, 192, 8)])
def test_dx_one_contraction_vs_fp64(pkg, ndir, R, C, N):
    """dX = dG_0 . W_0 + dG_1 . W_1 as one f16x3 GEMM over K = ndir * Kp, within the bound of the f16x3 GEMM tests."""
    ops = pkg.ops
    torch.manual_seed(R + N)
    g = torch.randn(ndir, R, C, device=DEV)
    ws = [torch.randn(C, N, device=DEV) * 0.05 for _ in range(ndir)]
    _, grow, _ = ops.f16_split_dg(g)
    out = ops.gemm_f16x3(grow, ops.f16_split_cat_t(ws, grow[0].shape[2] // ndir))
    ref = sum(g[d].double() @ ws[d].double() for d in range(ndir))
    sg = sum(_sgemm(g[d], ws[d]) for d in range(ndir))
    e, es = _err(out, ref), _err(sg, ref)
    assert e < 3e-6 and e <= 20 * max(es, 2.0 ** -24), (e, es)


@pytest.mark.parametrize("B,T,I,H", [(64, 1198, 120, 512), (64, 599, 2048, 512), (32, 299, 640, 640)])
def test_bilstm_full_size_vs_fp64(pkg, B, T, I, H):
    """BASELINE sizes (cfg B/C layer 0 and layer 1, cfg D): forward outputs, input gradient and every weight gradient
    of the f16x3 layer path against a float64 LSTM."""
    torch.manual_seed(3)
    ref = torch.nn.LSTM(I, H, bidirectional=True, num_layers=1, batch_first=True).to(DEV).double()
    torch.manual_seed(4)
    x = torch.randn(B, T, I, device=DEV)
    xr = x.double().requires_grad_(True)
    with torch.backends.cudnn.flags(enabled=False):
        yr, _ = ref(xr)
        gy = torch.randn(yr.shape, device=DEV)
        yr.backward(gy.double())
    params = [p.detach().float().requires_grad_(True) for p in ref.parameters()]
    xg = x.clone().requires_grad_(True)
    y = pkg.ops.bilstm(xg, params, 2)
    assert scaled_err(y.detach().cpu().numpy(), yr.detach().cpu().numpy()) < 2e-5
    y.backward(gy)
    assert scaled_err(xg.grad.cpu().numpy(), xr.grad.cpu().numpy()) < 1e-4
    for p, q, (name, _) in zip(params, ref.parameters(), ref.named_parameters()):
        scale = float(q.grad.abs().max())
        assert float((p.grad.double() - q.grad).abs().max()) < 5e-4 * max(scale, 1e-3), name
