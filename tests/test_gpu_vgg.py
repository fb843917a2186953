"""VGGExtractor on the GPU path (ops.VGGFn: conv-mode 3xTF32 GEMM + csrc/vgg.cu) against the float64 restatement
oracle/vgg_ref.py.

Forward, per conv.  Each conv is checked on its own input as the GPU saved it, so errors do not compound: with
a = the float64 conv of that input, S = the float64 conv of |input| with |w|, K = 9 C (32 for the first conv's
im2col), KB = K / 32 and chunks = ceil(KB / 4) + 1, the 3xTF32 bound of tests/test_host_gemm_bounds.py (_bound, one
slice) is
    bound = (3 2^-20 + 2 2^-23 12 4) S + (chunks + 3) 2^-24 (S + |bias|) + 2^-100.
The GPU stores relu(a_gpu) with |a_gpu - a| <= bound, and ReLU is 1-Lipschitz: |y_gpu - relu(a)| <= bound.  Max-pool
outputs and window indices must equal ATen's max_pool2d_with_indices of the GPU's own activation, bit for bit.

Forward, end to end.  e1 = bound1; e_{l+1} = conv(e_l, |w_{l+1}|) + bound_{l+1} (the conv of the error plus the new
rounding), through max-pool as maxpool(e) (|max a - max b| <= max |a - b|); |out - out64| <= e_out.

Gradients.  The float64 backward takes the GPU's own conv inputs, ReLU masks and pool choices (vgg_ref.routed_backward);
A = the same backward on absolute values (|dout|, |w|, |inputs|) bounds every sum of terms.  Every contraction of the
backward chain (three input gradients, four weight gradients over up to R grid rows) adds at most
eps = 3 2^-20 + 96 2^-23 + (R / 128 + 40) 2^-24 of its terms' absolute sum, and an error in dY reaches the weight and
bias gradients through no more than four of them: |g - g64| <= 4 eps A + 2^-100.  Separately, the GPU's masks and pool
choices equal float64's wherever the float64 pre-activation (or the gap between a window's two largest values) is
larger than the forward's propagated error.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import vgg_ref as V

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _module(pkg, cin, Fq, seed, bias=0.1):
    """VGGExtractor on the GPU; biases uniform in [-bias, bias] for bias > 0, zero for 0, and positive, uniform in
    [0.05, -bias], for bias < 0."""
    torch.manual_seed(seed)
    m = pkg.module.VGGExtractor(cin * Fq)
    with torch.no_grad():
        for i in (0, 2, 5, 7):
            if bias == 0:
                m.extractor[i].bias.zero_()
            else:
                m.extractor[i].bias.uniform_(-bias, bias) if bias > 0 else m.extractor[i].bias.uniform_(0.05, -bias)
    return m.to(DEV)


def _params(m):
    ps = []
    for i in (0, 2, 5, 7):
        ps += [m.extractor[i].weight, m.extractor[i].bias]
    return ps


def _features(B, T_in, cin, Fq, seed, lens=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T_in, cin * Fq, generator=g)
    if lens is not None:
        for b, n in enumerate(lens):
            x[b, n:] = 0
    return x.to(DEV)


def _gpu_state(out, B, T, Fq):
    """The GPU's saved conv inputs [x, y1, p1, y3], activations [y1..y4] and pool indices, as float64 [B, C, T, F]."""
    x0, y1, y2, p1, y3, y4, i1, i2 = out.grad_fn.saved_tensors[:8]
    T2, F2 = T // 2, Fq // 2
    up = lambda buf, t, f: V.unpad(buf, B, t, f).double()
    acts = [up(y1, T, Fq), up(y2, T, Fq), up(y3, T2, F2), up(y4, T2, F2)]
    return acts, up(p1, T2, F2), (i1.permute(0, 3, 1, 2).long(), i2.permute(0, 3, 1, 2).long())


def _bound(S, bias, K):
    KB = -(-K // 32)
    chunks = -(-KB // 4) + 1
    return (3 * 2.0 ** -20 + 2 * 2.0 ** -23 * 12 * 4) * S + (chunks + 3) * 2.0 ** -24 * (S + bias.abs()[None, :, None, None]) \
        + 2.0 ** -100


def _conv_check(inp, w, b, y_gpu, K):
    """Per-element forward bound of one conv on the GPU's own input; returns (bound, float64 pre-activation)."""
    a = F.conv2d(inp, w, b, padding=1)
    bnd = _bound(F.conv2d(inp.abs(), w.abs(), padding=1), b, K)
    err = (y_gpu - torch.relu(a)).abs()
    assert bool((err <= bnd).all()), float((err / bnd).max())
    return bnd, a


def _aten_indices(y, window_idx):
    """(ATen's flat indices of max_pool2d_with_indices on y, the GPU's window indices as flat indices)."""
    _, ai = F.max_pool2d(y.float(), 2, 2, return_indices=True)
    T2, F2 = window_idx.shape[2], window_idx.shape[3]
    Fq = y.shape[3]
    t2 = torch.arange(T2, device=y.device)[:, None]
    f2 = torch.arange(F2, device=y.device)[None, :]
    gi = (2 * t2 + window_idx // 2) * Fq + 2 * f2 + window_idx % 2
    return ai, gi


def _run_and_check(pkg, cin, Fq, B, T_in, seed, lens=None, bias=0.1, need_dx=True, device64="cpu"):
    m = _module(pkg, cin, Fq, seed, bias)
    feat = _features(B, T_in, cin, Fq, seed + 1, lens).requires_grad_(need_dx)
    flen = torch.full((B,), T_in, device=DEV)
    out, olen = m(feat, flen)
    T = T_in - T_in % 4
    T2, F2 = T // 2, Fq // 2
    assert out.shape == (B, T // 4, 128 * (F2 // 2)) and torch.equal(olen, flen // 4)
    (y1, y2, y3, y4), p1, (i1, i2) = _gpu_state(out, B, T, Fq)
    ps = [p.detach().double() for p in _params(m)]
    ps64 = [p.to(device64) for p in ps]
    x = V.view_input(feat.detach().double(), cin)
    dv = lambda t: t.to(device64)
    # per conv, on the GPU's own input
    b1, a1 = _conv_check(dv(x), ps64[0], ps64[1], dv(y1), 32)
    b2, a2 = _conv_check(dv(y1), ps64[2], ps64[3], dv(y2), 9 * 64)
    b3, a3 = _conv_check(dv(p1), ps64[4], ps64[5], dv(y3), 9 * 64)
    b4, a4 = _conv_check(dv(y3), ps64[6], ps64[7], dv(y4), 9 * 128)
    # max-pool: values and indices as ATen's on the GPU's activations
    for y, idx, pooled in ((y2, i1, p1), (y4, i2, None)):
        ai, gi = _aten_indices(y, idx)
        assert torch.equal(ai, gi)
        ref = F.max_pool2d(y, 2, 2)
        got = pooled if pooled is not None else out.detach().double().view(B, T // 4, 128, F2 // 2).transpose(1, 2)
        assert torch.equal(torch.isnan(got), torch.isnan(ref)) and torch.equal(got.nan_to_num(), ref.nan_to_num())
    # end to end against float64 with the propagated bound
    r = V.forward(feat, cin, ps, device=device64)
    e1 = b1
    e2 = F.conv2d(e1, ps64[2].abs(), padding=1) + b2
    e3 = F.conv2d(F.max_pool2d(e2, 2, 2), ps64[4].abs(), padding=1) + b3
    e4 = F.conv2d(e3, ps64[6].abs(), padding=1) + b4
    e_out = V.flatten_output(F.max_pool2d(e4, 2, 2))
    err = (out.detach().double().to(device64) - r["out"]).abs()
    assert bool((err <= e_out).all()), float((err / e_out).max())
    # masks and pool choices against float64: different only within the propagated error
    for y, a, e in ((y1, r["a1"], e1), (y2, r["a2"], e2), (y3, r["a3"], e3), (y4, r["a4"], e4)):
        differ = dv(~(y <= 0)) != (a > 0)
        assert bool((a[differ].abs() <= e[differ]).all())
    for idx, yref, e in ((i1, r["y2"], e2), (i2, r["y4"], e4)):
        T2_, F2_ = idx.shape[2], idx.shape[3]
        win = torch.stack([yref[:, :, k // 2:2 * T2_:2, k % 2:2 * F2_:2] for k in range(4)], -1)
        ew = torch.stack([e[:, :, k // 2:2 * T2_:2, k % 2:2 * F2_:2] for k in range(4)], -1)
        picked = win.gather(-1, dv(idx)[..., None])[..., 0]
        assert bool((win.max(-1).values - picked <= 2 * ew.max(-1).values).all())
    # gradients against the routed float64 backward
    dout = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed + 2)).to(DEV)
    out.backward(dout)
    inputs = [dv(x), dv(y1), dv(p1), dv(y3)]
    masks = [dv(~(y <= 0)) for y in (y1, y2, y3, y4)]
    idx64 = (dv(i1), dv(i2))
    g64, dx64 = V.routed_backward(inputs, masks, idx64, ps64, dout, need_dx)
    gabs, dxabs = V.routed_backward([t.abs() for t in inputs], masks, idx64, [p.abs() for p in ps64], dout.abs(),
                                    need_dx)
    R = B * (T + 2) * (Fq + 2)
    eps = 3 * 2.0 ** -20 + 96 * 2.0 ** -23 + (R / 128 + 40) * 2.0 ** -24
    for p, g, a in zip(_params(m), g64, gabs):
        err = (p.grad.double().to(device64) - g).abs()
        assert bool((err <= 4 * eps * a + 2.0 ** -100).all()), float((err / (4 * eps * a + 2.0 ** -100)).max())
    if need_dx:
        gx = V.view_input(feat.grad.double(), cin).to(device64)
        err = (gx - dx64).abs()
        assert bool((err <= 4 * eps * dxabs + 2.0 ** -100).all())
        assert not bool(feat.grad[:, T:].any())
    return m, feat, out, r


SWEEP = [(cin, Fq, r) for cin in (1, 2, 3) for Fq in (40, 13) for r in range(4)]


@pytest.mark.parametrize("cin,Fq,rem", SWEEP)
def test_shape_sweep_matches_float64(pkg, cin, Fq, rem):
    """Ragged lengths (zero frames past each end), B = 3 (65+ M tiles of 128 rows at F = 40; every weight gradient
    split along K), T mod 4 = rem."""
    B, T_in = 3, 64 + rem
    _run_and_check(pkg, cin, Fq, B, T_in, seed=10 * cin + Fq + rem, lens=[T_in, T_in - 9, T_in - 30],
                   need_dx=(rem % 2 == 0))


def test_full_size_example_shape(pkg):
    """The reference example's shape: B = 16, T = 1196, C_in = 3, F = 40 (float64 on the device)."""
    lens = [1196 - 37 * b for b in range(16)]
    _run_and_check(pkg, 3, 40, 16, 1196, seed=3, lens=lens, need_dx=False, device64=DEV)


def test_grid_operands_make_the_first_two_convs_exact(pkg):
    """Integer features |x| <= 7, weights |w| <= 7 and biases |b| <= 64 (tests/test_gpu_gemm_parity.py's exact grid):
    2^0 (sum |x w| + |b|) < 2^24 holds for conv1 (K = 27) and conv2 (K = 576, checked below), so both convs are
    bit-equal to float64; a wrong tap, shift or junk row changes a value."""
    from test_gpu_gemm_parity import grid_operand, grid_extra
    cin, Fq, B, T_in = 3, 40, 2, 48
    g = torch.Generator(device=DEV).manual_seed(4)
    m = _module(pkg, cin, Fq, 1)
    with torch.no_grad():
        for i in (0, 2):
            w = m.extractor[i].weight
            w.copy_(grid_operand("int", w.shape[0], w[0].numel(), g).view_as(w))
            m.extractor[i].bias.copy_(grid_extra("int", (w.shape[0],), g))
    feat = grid_operand("int", B * T_in, cin * Fq, g).view(B, T_in, cin * Fq)
    out, _ = m(feat, torch.full((B,), T_in, device=DEV))
    (y1, y2, _, _), _, _ = _gpu_state(out, B, T_in, Fq)
    r = V.forward(feat, cin, [p.detach() for p in _params(m)])
    for y, ref, inp, wi in ((y1, r["y1"], r["x"], 0), (y2, r["y2"], r["y1"], 2)):
        w = m.extractor[wi].weight.detach().double().cpu()
        S = F.conv2d(inp.abs(), w.abs(), padding=1) + m.extractor[wi].bias.detach().double().cpu().abs()[None, :, None, None]
        assert float(S.max()) < 2 ** 24
        assert torch.equal(y.cpu(), ref)


def test_zero_receptive_field_gives_exact_zeros(pkg):
    """Zero biases (the Adadelta init): every activation whose receptive field is all zero is exactly 0 and its ReLU
    mask is closed, so no gradient passes there (the reason the path does not use transform-domain convolutions)."""
    cin, Fq, B, T_in = 1, 40, 3, 80
    m = _module(pkg, cin, Fq, 5, bias=0)
    feat = _features(B, T_in, cin, Fq, 6, lens=[80, 41, 17])
    out, _ = m(feat, torch.full((B,), T_in, device=DEV))
    acts, _, _ = _gpu_state(out, B, T_in, Fq)
    ra = V.forward(feat.abs(), cin, [p.detach().abs() for p in _params(m)])
    zeros = 0
    for y, key in zip(acts, ("y1", "y2", "y3", "y4")):
        rf0 = ra[key].to(DEV) == 0
        zeros += int(rf0.sum())
        assert bool((y[rf0] == 0).all()) and not bool((~(y[rf0] <= 0)).any())
    assert zeros > 0
    rp = ra["out"].to(DEV) == 0
    assert bool((out.detach()[rp] == 0).all())
    _run_and_check(pkg, cin, Fq, B, T_in, seed=5, lens=[80, 41, 17], bias=0)


def test_ties_and_nan_route_as_aten(pkg):
    """Positive biases make every window past an utterance's end constant (ties: the first element wins); NaN features
    reach the pools as NaN (the last NaN of a window wins).  Both route exactly as max_pool2d_with_indices."""
    _run_and_check(pkg, 2, 13, 3, 72, seed=8, lens=[72, 50, 23], bias=-0.3)
    cin, Fq, B, T_in = 1, 40, 2, 40
    m = _module(pkg, cin, Fq, 9, bias=-0.3)
    feat = _features(B, T_in, cin, Fq, 10, lens=[40, 20])
    feat[0, 5, 7] = float("nan")
    feat[1, 30, 2] = float("nan")
    out, _ = m(feat, torch.full((B,), T_in, device=DEV))
    acts, p1, (i1, i2) = _gpu_state(out, B, T_in, Fq)
    assert bool(torch.isnan(acts[3]).any())
    for y, idx in ((acts[1], i1), (acts[3], i2)):
        ai, gi = _aten_indices(y, idx)
        assert torch.equal(ai, gi)


def test_fewer_than_four_frames_raise_before_any_launch(pkg):
    m = _module(pkg, 1, 40, 0)
    feat = torch.randn(2, 3, 40, device=DEV)
    torch.cuda.synchronize()
    n0 = pkg.lib.launch_count()
    with pytest.raises(ValueError, match="at least 4 frames"):
        m(feat, torch.tensor([3, 2], device=DEV))
    assert pkg.lib.launch_count() == n0


def test_no_library_convolution_pooling_or_relu(pkg, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("library op called on the CUDA VGG path")
    for mod, name in ((F, "conv2d"), (F, "max_pool2d"), (F, "relu"), (torch, "relu"), (torch, "conv2d"),
                      (torch, "max_pool2d"), (F, "max_pool2d_with_indices"), (torch, "convolution")):
        monkeypatch.setattr(mod, name, refuse)
    m = _module(pkg, 3, 40, 2)
    feat = _features(2, 45, 3, 40, 3).requires_grad_(True)
    out, _ = m(feat, torch.tensor([45, 30], device=DEV))
    out.square().sum().backward()
    assert torch.isfinite(feat.grad).all() and all(p.grad is not None for p in m.parameters())


def test_cuda_graph_replay_equals_eager_steps_vgg(pkg):
    """Whole-step CUDA graph of a tiny `prenet: vgg` model: replays reproduce the eager train steps."""
    from test_gpu_model import _tiny_config
    cfg = _tiny_config("vgg")
    g = torch.Generator().manual_seed(11)
    wave = torch.clamp(0.05 * torch.randn(3, 9000, generator=g), -1, 1).to(DEV)
    lens = torch.tensor([9000, 9000, 9000], device=DEV)
    txt = torch.tensor([[3, 4, 4, 5, 1], [6, 7, 1, 0, 0], [8, 9, 10, 1, 0]], device=DEV)
    eager = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    graph = pkg.TrainStep(cfg, 12, device=DEV, seed=5)
    for _ in range(3):
        eager(wave, lens, txt, max_len=5)
    assert graph.capture(wave, lens, txt, warmup=3), graph.graph_error
    for it in range(3):
        le = eager(wave * (1.0 - 0.1 * it), lens, txt, max_len=5)
        lg = graph(wave * (1.0 - 0.1 * it), lens, txt)
        assert abs(le.item() - lg.item()) <= 1e-6 * abs(le.item()), (it, le.item(), lg.item())
    for (k, a), (_, b) in zip(eager.model.state_dict().items(), graph.model.state_dict().items()):
        assert float((a - b).abs().max()) <= 1e-6 * max(float(a.abs().max()), 1e-3), k
