"""The GRU encoder layer on the persistent recurrence kernels: b200asr_bigru_fwd / _bwd through the C ABI against the
float64 recurrence of oracle/gruenc_ref, RNNLayer(module='GRU') against float64 / ATen nn.GRU, its routing, the
model_gruenc golden and CUDA-graph replay of a GRU-encoder train step.

The GRU runs on the BiLSTM's kernels with another pointwise cell (csrc/rnn_cell.cuh): same dispatcher, same variants.
So every case asserts the variant it reaches through b200asr_debug_lstm_variant, and the parity cases are those of
tests/test_gpu_lstm_variants.py, which together reach every code path the sweep of the query reaches.

Bounds, per batch row and relative to the row's own largest float64 value (EPS = 2^-24), fixed here:
    err_kernel(row) <= K * max(err_fp32(row), FLOOR),   K = 8,   FLOOR = 16 * EPS
  * err_fp32 is the error of the same GRU recurrence run in float32 on the CPU (gruenc_ref.recurrence) against the
    float64 one, computed in the test: it carries the conditioning of the recurrence at these inputs.
  * The kernels differ from that float32 loop only in the step products h . W_hh^T and dG . W_hh (operands of about
    22 significant bits instead of 24, DESIGN.md section 4: a product rounding at most 4x that of fp32, accumulated in
    another order): K = 8 is that 4x with a factor 2 for the summation order, as for the LSTM.
  * FLOOR covers rows the float32 loop gets almost exactly (T = 1 has no product): the GRU cell is two sigmoids and a
    tanh (within 2 ulp each) and five rounded adds / multiplies per step forward, about 10 ulp; 16 ulp of the row scale.
tests/test_host_gru_encoder.py shows on the CPU that this bound accepts an fp32 emulation of the kernels' cell and
rejects planted cell defects by at least 10x.
"""
import pytest
import torch

import test_gpu_lstm_variants as V
from oracle import gruenc_ref, lstm_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _inputs(B, T, H, ndir, seed, wscale=1.0):
    """test_gpu_lstm_variants' inputs (pre-activations with a fraction at +-30, an all-zero row 0, dout rows at 2^k,
    an all-zero dout row 1) with W_hh in the packed GRU layout: slot 2 (gi_n) has no hidden product."""
    pre, whh, dout = V._inputs(B, T, H, ndir, seed, wscale)
    whh.view(ndir, 4, H, H)[:, 2] = 0.0
    return pre, whh, dout


def _run(pkg, pre, whh, dout, mode):
    """b200asr_bigru_fwd then _bwd under debug `mode`: (out, hstate, activated-gate stash, dG) on the CPU.  The outputs
    the calls must write start as NaN."""
    L = pkg.lib
    lib = pkg.load_library()
    ndir, B, T, H, _ = pre.shape
    gates = pre.to(DEV).contiguous()
    w = whh.to(DEV).contiguous()
    hst = torch.full((ndir, B, T, H), float("nan"), device=DEV)
    out = torch.full((B, T, ndir * H), float("nan"), device=DEV)
    lib.b200asr_debug_set_lstm_mode(mode)
    try:
        nbytes = lib.b200asr_bilstm_workspace_bytes(B, T, H, ndir)
        ws = torch.empty(nbytes, device=DEV, dtype=torch.uint8)
        L.check(lib.b200asr_bigru_fwd(L.ptr(gates), L.ptr(w), L.ptr(hst), L.ptr(out), B, T, H, ndir, L.ptr(ws),
                                      nbytes, L.stream()), "bigru_fwd")
        stash = gates.clone()
        dd = dout.to(DEV).contiguous()
        L.check(lib.b200asr_bigru_bwd(L.ptr(gates), L.ptr(w), L.ptr(hst), L.ptr(dd), B, T, H, ndir, L.ptr(ws),
                                      nbytes, L.stream()), "bigru_bwd")
    finally:
        lib.b200asr_debug_set_lstm_mode(0)
    return out.cpu(), hst.cpu(), stash.cpu(), gates.cpu()


def _parity(pkg, B, H, ndir, mode, T, seed, wscale=1.0, pre_nan=None, dout_nan=None, twice=True):
    pre, whh, dout = _inputs(B, T, H, ndir, seed, wscale)
    if pre_nan is not None:
        b, t = pre_nan
        pre[0, b, t, H // 3, 1] = float("nan")
    if dout_nan is not None:
        b, t = dout_nan
        dout[b, t, H // 2] = float("nan")
    got = _run(pkg, pre, whh, dout, mode)
    r64 = gruenc_ref.recurrence(pre, whh, dout, torch.float64)
    r32 = gruenc_ref.recurrence(pre, whh, dout, torch.float32)
    res = V._check_rows(got, r64, r32, ("GRU", B, H, ndir, mode, T))
    if twice:
        again = _run(pkg, pre, whh, dout, mode)
        for name, a, b in zip(V.NAMES, got, again):
            assert torch.equal(V._bits(a), V._bits(b)), (name, "differs between two runs")
    return res


# ------------------------------------------------------------------------------------------- every variant
@pytest.mark.parametrize("B,H,ndir,mode,T,fwd,bwd", V.CASES, ids=V._ids(V.CASES))
def test_gru_recurrence_vs_fp64_per_row(pkg, B, H, ndir, mode, T, fwd, bwd):
    assert V._labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    ratio, err = _parity(pkg, B, H, ndir, mode, T, seed=B * 7 + H + mode + 1)
    print("GRU %s | %s: worst row error %.3g (%.3g of the bound)" % (fwd, bwd, err, ratio))


@pytest.mark.parametrize("T", [1, 2, 3, 4, 5, 9, 17])
@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", V.EDGE_SHAPES, ids=[str(s[3]) for s in V.EDGE_SHAPES])
def test_gru_time_edges(pkg, B, H, ndir, mode, fwd, bwd, T):
    assert V._labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    _parity(pkg, B, H, ndir, mode, T, seed=200 + T, twice=False)


@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", V.EDGE_SHAPES, ids=[str(s[3]) for s in V.EDGE_SHAPES])
def test_gru_long_sequence(pkg, B, H, ndir, mode, fwd, bwd):
    assert V._labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    ratio, err = _parity(pkg, B, H, ndir, mode, 300, seed=8, twice=False)
    print("GRU T = 300 %s | %s: worst row error %.3g (%.3g of the bound)" % (fwd, bwd, err, ratio))


@pytest.mark.parametrize("B,H,ndir,mode,fwd,bwd", V.EDGE_SHAPES, ids=[str(s[3]) for s in V.EDGE_SHAPES])
def test_gru_nan_stays_in_its_row(pkg, B, H, ndir, mode, fwd, bwd):
    """A NaN pre-activation in row 3 at frame 4 and a NaN dout in row 6 at frame 2."""
    assert V._labels(pkg.load_library(), B, H, ndir, mode) == (fwd, bwd)
    _parity(pkg, B, H, ndir, mode, 9, seed=14, pre_nan=(3, 4), dout_nan=(6, 2), twice=False)


# ------------------------------------------------------------------------------------------- wgmma backward clusters
CAP_MODES = {1: 16, 2: 32, 4: 0}          # debug lstm mode word that caps the backward's cluster size at CS


def _cluster(lib, B, H, ndir, mode):
    lib.b200asr_debug_set_lstm_mode(mode)
    try:
        return lib.b200asr_debug_lstm_cluster(B, H, ndir, 1)
    finally:
        lib.b200asr_debug_set_lstm_mode(0)


@pytest.mark.parametrize("B,H,ndir,T", [(64, 512, 2, 17), (64, 256, 2, 9), (32, 640, 2, 5)])
def test_gru_every_cluster_size_vs_fp64(pkg, B, H, ndir, T):
    """Every cluster size the planner takes for the shape (and CS = 1 through the cap); forward outputs bit-equal."""
    lib = pkg.load_library()
    reach = {}
    for cs, mode in sorted(CAP_MODES.items()):
        got = _cluster(lib, B, H, ndir, mode)
        assert 1 <= got <= cs
        reach.setdefault(got, mode)
    assert 1 in reach
    fwd = None
    for cs, mode in sorted(reach.items()):
        assert V._labels(lib, B, H, ndir, mode)[1].startswith("wgmma")
        ratio, err = _parity(pkg, B, H, ndir, mode, T, seed=B + H + T, dout_nan=(3, T // 2))
        print("GRU CS=%d: worst row error %.3g (%.3g of the bound)" % (cs, err, ratio))
        got = _run(pkg, *_inputs(B, T, H, ndir, seed=B + H + T), mode)
        if fwd is None:
            fwd = got[:3]
        else:
            for name, a, b in zip(V.NAMES, fwd, got[:3]):
                assert torch.equal(V._bits(a), V._bits(b)), (name, "forward differs between cluster sizes", cs)


def test_gru_cfg_b_reaches_clusters(pkg):
    assert _cluster(pkg.load_library(), 64, 512, 2, 0) in (2, 4)


# ------------------------------------------------------------------------------------------- the layer
def _nn_gru_grads(ref, x, gy, dt):
    m = ref if dt == torch.float32 else _clone_gru(ref, dt)
    xr = x.clone().to(dt).requires_grad_(True)
    y, _ = m(xr)
    y.backward(gy.to(dt))
    return [y.detach(), xr.grad] + [p.grad for p in m.parameters()]


def _clone_gru(ref, dt):
    m = torch.nn.GRU(ref.input_size, ref.hidden_size, bidirectional=ref.bidirectional, batch_first=True).to(dt)
    m.load_state_dict({k: v.to(dt) for k, v in ref.state_dict().items()})
    return m


def _layer(pkg, ref, I, H):
    layer = pkg.module.RNNLayer(I, "GRU", H, True, 0, False, 1, "drop", False)
    layer.layer.load_state_dict(ref.state_dict())
    return layer.to(DEV)


@pytest.mark.parametrize("I", [40, 42])
@pytest.mark.parametrize("mode,fwd", [(0, "wgmma8/flag/vec"), (3, "mma.sync/v2"), (1, "fma1x4")])
def test_rnn_layer_gru_vs_fp64_nn_gru(pkg, mode, fwd, I):
    """RNNLayer(module='GRU') forward + backward once per generation, for an input width on the f16x3 layer GEMMs
    (I % 4 == 0) and one on the Split path: out, dx and the four parameter gradients of each direction against
    nn.GRU in float64, per tensor, within K times nn.GRU's float32 error."""
    B, T, H = 32, 12, 256
    lib = pkg.load_library()
    assert lstm_ref.label(lstm_ref.variant(lib, B, H, 2, False, mode), False) == fwd
    torch.manual_seed(22 + I)
    ref = torch.nn.GRU(I, H, bidirectional=True, batch_first=True)
    x = torch.randn(B, T, I)
    x[5, 7:] = 0.0                                              # a ragged, zero-padded utterance
    gy = torch.randn(B, T, 2 * H)
    r64 = _nn_gru_grads(ref, x, gy, torch.float64)
    r32 = _nn_gru_grads(ref, x, gy, torch.float32)
    layer = _layer(pkg, ref, I, H)
    xg = x.to(DEV).requires_grad_(True)
    lib.b200asr_debug_set_lstm_mode(mode)
    try:
        y, _ = layer(xg, torch.full((B,), T))
        y.backward(gy.to(DEV))
    finally:
        lib.b200asr_debug_set_lstm_mode(0)
    got = [y.detach().cpu(), xg.grad.cpu()] + [p.grad.cpu() for p in layer.layer.parameters()]
    names = ["out", "dx"] + [n for n, _ in ref.named_parameters()]
    for name, k, r, f in zip(names, got, r64, r32):
        scale = float(r.abs().max())
        ek = float((k.double() - r).abs().max()) / scale
        ef = float((f.double() - r).abs().max()) / scale
        assert ek <= V.K * max(ef, V.FLOOR), (name, ek, ef)


@pytest.mark.parametrize("B,T,I,H", [(64, 1198, 120, 512), (64, 599, 2048, 512)])
def test_rnn_layer_gru_full_size_vs_aten_cpu(pkg, B, T, I, H):
    """The cfg-B encoder layer shapes over all 1198 / 599 steps against ATen's CPU GRU in fp32, with the BiLSTM
    full-size tolerances (tests/test_gpu_kernels.py): output, input gradient and every weight gradient."""
    torch.set_num_threads(16)
    torch.manual_seed(3)
    ref = torch.nn.GRU(I, H, bidirectional=True, batch_first=True)
    torch.manual_seed(4)
    x = torch.randn(B, T, I)
    xr = x.clone().requires_grad_(True)
    yr, _ = ref(xr)
    gy = torch.randn_like(yr)
    yr.backward(gy)
    layer = _layer(pkg, ref, I, H)
    xg = x.to(DEV).requires_grad_(True)
    y, _ = layer(xg, torch.full((B,), T))
    y.backward(gy.to(DEV))
    from conftest import scaled_err
    assert scaled_err(y.detach().cpu().numpy(), yr.detach().numpy()) < 2e-5
    assert scaled_err(xg.grad.cpu().numpy(), xr.grad.numpy()) < 1e-4
    for p, q, (name, _) in zip(layer.layer.parameters(), ref.parameters(), ref.named_parameters()):
        scale = float(q.grad.abs().max())
        assert float((p.grad.cpu() - q.grad).abs().max()) < 5e-4 * max(scale, 1e-3), name


def test_cuda_gru_layer_does_not_call_nn_gru(pkg, monkeypatch):
    """A CUDA GRU layer with a plan runs on the kernels (nn.GRU.forward would raise); H = 30 has no plan and still
    runs on nn.GRU, matching it."""
    def refuse(*a, **k):
        raise AssertionError("nn.GRU.forward called")
    torch.manual_seed(5)
    ref = torch.nn.GRU(24, 32, bidirectional=True, batch_first=True)
    layer = _layer(pkg, ref, 24, 32)
    x = torch.randn(3, 7, 24)
    with monkeypatch.context() as m:
        m.setattr(torch.nn.GRU, "forward", refuse)
        y, _ = layer(x.to(DEV), torch.full((3,), 7))
    yr, _ = ref(x)
    assert float((y.detach().cpu() - yr.detach()).abs().max()) < 1e-5
    ref30 = torch.nn.GRU(24, 30, bidirectional=True, batch_first=True)
    layer30 = _layer(pkg, ref30, 24, 30)
    assert not pkg.ops.rnn_layer_supported(3, 7, 30, 2)
    y30, _ = layer30(x.to(DEV), torch.full((3,), 7))
    y30r, _ = ref30(x)
    assert float((y30.detach().cpu() - y30r.detach()).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------- train step
def test_gru_encoder_cuda_graph_replay_equals_eager_steps(pkg):
    """Whole-step CUDA graph replays of a model with a 2-layer GRU encoder reproduce the eager train steps."""
    from test_gpu_model import _tiny_config
    cfg = _tiny_config("hybrid")
    cfg["model"]["encoder"] = dict(cfg["model"]["encoder"], module="GRU")
    g = torch.Generator().manual_seed(12)
    wave = torch.clamp(0.05 * torch.randn(3, 9000, generator=g), -1, 1).to(DEV)
    lens = torch.tensor([9000, 9000, 9000], device=DEV)
    txt = torch.tensor([[3, 4, 4, 5, 1], [6, 7, 1, 0, 0], [8, 9, 10, 1, 0]], device=DEV)
    eager = pkg.TrainStep(cfg, 12, device=DEV, seed=6)
    graph = pkg.TrainStep(cfg, 12, device=DEV, seed=6)
    assert isinstance(eager.model.encoder.layers[0].layer, torch.nn.GRU)
    for _ in range(2):
        eager(wave, lens, txt, max_len=5)
    assert graph.capture(wave, lens, txt, warmup=2), graph.graph_error
    for it in range(2):
        le = eager(wave * (1.0 - 0.1 * it), lens, txt, max_len=5)
        lg = graph(wave * (1.0 - 0.1 * it), lens, txt)
        assert le.item() == lg.item(), (it, le.item(), lg.item())
    for (k, a), (_, b) in zip(eager.model.state_dict().items(), graph.model.state_dict().items()):
        assert torch.equal(a, b), k


# ------------------------------------------------------------------------------------------- golden model
def test_gruenc_golden_model_matches_reference(pkg, monkeypatch):
    """model_gruenc (oracle/make_golden_gruenc.py: the reference with a 2-layer bidirectional GRU encoder, layer 0 on
    the wgmma step kernels) through ASR: outputs, losses, every gradient and greedy ids, with the tolerances of
    test_gpu_model.test_train_step_matches_reference / test_greedy_inference_ids_bit_exact."""
    import test_gpu_model as M
    from oracle.make_golden_gruenc import SPEC, gruenc_model_cfg
    lib = pkg.load_library()
    B, H = SPEC[2], gruenc_model_cfg()["encoder"]["dim"][0]
    assert V._labels(lib, B, H, 2, 0) == ("wgmma8/flag/vec", "wgmma8/poll")
    base = M.tiny_model_cfg
    monkeypatch.setattr(M, "tiny_model_cfg", lambda kind: gruenc_model_cfg() if kind == "gruenc" else base(kind))
    M.test_train_step_matches_reference(pkg, "gruenc")
    M.test_greedy_inference_ids_bit_exact(pkg, "gruenc")
