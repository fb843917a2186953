"""Per-step time of the BiLSTM step-kernel families (wgmma / mma.sync 3xTF32 / packed fp32 FMA) at one shape.
   env: B (64), H (512), T (300), I (1024).  Prints us/step for forward and backward and the max |difference| of the
   outputs / input gradients between the two families."""
import importlib, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")
L = pkg.lib
B, H, T, I = (int(os.environ.get(k, d)) for k, d in (("B", 64), ("H", 512), ("T", 300), ("I", 1024)))
torch.manual_seed(0)
ref = torch.nn.LSTM(I, H, bidirectional=True, batch_first=True)
params = [p.detach().cuda().requires_grad_(True) for p in ref.parameters()]
x = torch.randn(B, T, I, device="cuda", requires_grad=True)
gy = torch.randn(B, T, 2 * H, device="cuda")
lib = L.load()
res = {}
MODES = ((3, "mma.sync"), (0, "wgmma"))
if os.environ.get("ONLY_MODES"):
    MODES = tuple(m for m in MODES if str(m[0]) in os.environ["ONLY_MODES"].split(","))
if os.environ.get("EXTRA_MODE"):
    MODES += ((int(os.environ["EXTRA_MODE"]), "wgmma-mode%s" % os.environ["EXTRA_MODE"]),)
REPS = int(os.environ.get("REPS", 3))
stats = {name: [] for _, name in MODES}
fwd_only = {name: [] for _, name in MODES}
for rep in range(REPS):
    for mode, name in MODES:
        lib.b200asr_debug_set_lstm_mode(mode)
        for it in range(3):
            if it == 1:
                L.TIMER.enabled = True
                L.TIMER.reset()
            x.grad = None
            y = pkg.ops.bilstm(x, params, 2)
            y.backward(gy)
        torch.cuda.synchronize()
        L.TIMER.enabled = False
        s = L.TIMER.summary()
        res[name] = (y.detach().clone(), x.grad.detach().clone())
        stats[name].append((1e3 * s["bilstm_fwd"]["ms"] / s["bilstm_fwd"]["launches"] / T,
                            1e3 * s["bilstm_bwd"]["ms"] / s["bilstm_bwd"]["launches"] / T))
        with torch.no_grad():                       # forward kernels back to back, no backward in between
            L.TIMER.enabled = True
            L.TIMER.reset()
            for it in range(3):
                pkg.ops.bilstm(x, params, 2)
            torch.cuda.synchronize()
            L.TIMER.enabled = False
            s = L.TIMER.summary()
            fwd_only[name].append(1e3 * s["bilstm_fwd"]["ms"] / s["bilstm_fwd"]["launches"] / T)
lib.b200asr_debug_set_lstm_mode(0)
for _, name in MODES:
    print("%-16s B=%d H=%d T=%d us/step: fwd %s | bwd %s | fwd alone %s" % (
        name, B, H, T, " ".join("%.2f" % f for f, _ in stats[name]), " ".join("%.2f" % b for _, b in stats[name]),
        " ".join("%.2f" % f for f in fwd_only[name])), flush=True)
a, b = res[MODES[0][1]], res[MODES[-1][1]]
print("max |dy| %.3e (max |y| %.3e)   max |d dx| %.3e (max |dx| %.3e)" % (
    float((a[0] - b[0]).abs().max()), float(a[0].abs().max()), float((a[1] - b[1]).abs().max()), float(a[1].abs().max())))
