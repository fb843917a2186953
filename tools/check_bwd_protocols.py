"""Full-size BiLSTM layer (B=64, T=1198, I=120, H=512): gradients of the three backward variants against each other
(default = wgmma + polling exchange, 2048 = wgmma + flag exchange, 512 = mma.sync generation) and, for scale,
against an fp64 CPU LSTM on the first rows.  Prints max-abs differences relative to each tensor's max."""
import importlib, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")
B, T, I, H = (int(os.environ.get(k, d)) for k, d in (("B", 64), ("T", 1198), ("I", 120), ("H", 512)))
torch.manual_seed(0)
ref = torch.nn.LSTM(I, H, bidirectional=True, batch_first=True)
x0 = torch.randn(B, T, I)
gy = torch.randn(B, T, 2 * H) * 0.01
lib = pkg.lib.load()
res = {}
for mode, name in ((0, "wgmma+poll"), (2048, "wgmma+flag"), (512, "mma.sync"), (0, "wgmma+poll again")):
    lib.b200asr_debug_set_lstm_mode(mode)
    params = [p.detach().cuda().requires_grad_(True) for p in ref.parameters()]
    x = x0.cuda().requires_grad_(True)
    y = pkg.ops.bilstm(x, params, 2)
    y.backward(gy.cuda())
    torch.cuda.synchronize()
    res[name] = [x.grad.double().cpu()] + [p.grad.double().cpu() for p in params]
lib.b200asr_debug_set_lstm_mode(0)
names = ["dx"] + [n for n, _ in ref.named_parameters()]
# fp64 reference
r64 = torch.nn.LSTM(I, H, bidirectional=True, batch_first=True).double()
r64.load_state_dict({k: v.double() for k, v in ref.state_dict().items()})
x64 = x0.double().requires_grad_(True)
torch.set_num_threads(32)
y64, _ = r64(x64)
y64.backward(gy.double())
res["fp64"] = [x64.grad] + [p.grad for p in r64.parameters()]
r32 = ref
x32 = x0.clone().requires_grad_(True)
y32, _ = r32(x32)
y32.backward(gy)
res["aten-cpu-fp32"] = [x32.grad.double()] + [p.grad.double() for p in r32.parameters()]
for a in ("wgmma+poll", "wgmma+flag", "mma.sync", "wgmma+poll again", "aten-cpu-fp32"):
    print("== %s vs fp64" % a)
    for n, u, v in zip(names, res[a], res["fp64"]):
        print("   %-28s %.3e" % (n, float((u - v).abs().max() / v.abs().max())))
    nu = sum(float((u ** 2).sum()) for u in res[a][1:]) ** 0.5
    nv = sum(float((v ** 2).sum()) for v in res["fp64"][1:]) ** 0.5
    print("   weight-grad norm rel err %.3e" % (abs(nu - nv) / nv))
