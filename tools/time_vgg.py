"""Time the VGG prenet's forward + backward on the GPU path (ops.VGGFn: conv-mode 3xTF32 GEMM + csrc/vgg.cu) against
the library sequence VGGExtractor ran before (nn.Conv2d / ReLU / MaxPool2d through ATen with cuDNN off, i.e. ATen's
direct convolution), alternating the two in one process.  Reports per shape the median and range of the step time
over repetitions, the achieved TFLOP/s from the algorithmic FLOP count (forward, input gradients of convs 2-4, weight
gradients), the per-kernel split of the GPU path (CUDA events per C-ABI call), the float64 parity of both paths, and
the card's name and power limit.

usage: python tools/time_vgg.py [--shapes 16x1196,64x1196] [--reps 7] [--iters 3] [--out result.json]"""
import argparse
import copy
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")

CIN, FQ = 3, 40


def flops(B, T, Fq, cin):
    """Algorithmic FLOPs of one train step of the prenet: forward + input gradients (convs 2-4) + weight gradients."""
    T2, F2 = T // 2, Fq // 2
    conv = [2 * 9 * T * Fq * cin * 64, 2 * 9 * T * Fq * 64 * 64, 2 * 9 * T2 * F2 * 64 * 128, 2 * 9 * T2 * F2 * 128 * 128]
    return B * (2 * sum(conv) + sum(conv[1:]))


def library_forward(m, feat, flen):
    x, _ = m.view_input(feat, flen)
    with torch.backends.cudnn.flags(enabled=False):
        y = m.extractor(x)
    y = y.transpose(1, 2)
    return y.contiguous().view(y.shape[0], y.shape[1], m.out_dim)


def step(path, m, feat, flen, dout):
    for p in m.parameters():
        p.grad = None
    out = m(feat, flen)[0] if path == "gpu" else library_forward(m, feat, flen)
    out.backward(dout)
    return out


def time_path(path, m, feat, flen, dout, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        step(path, m, feat, flen, dout)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def parity(path, m, feat, flen, dout, ref_out):
    out = step(path, m, feat, flen, dout).detach().double()
    torch.cuda.synchronize()
    res = {"out_max_abs_err_over_max_abs": float((out - ref_out).abs().max() / ref_out.abs().max())}
    return res, {k: p.grad.detach().double().clone() for k, p in m.named_parameters()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="16x1196,64x1196", help="BxT list")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_vgg.py measures on a GPU"
    dev = torch.device("cuda")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    result = {"card": smi[0] if smi else torch.cuda.get_device_name(), "shapes": []}
    for shape in args.shapes.split(","):
        B, T = (int(v) for v in shape.split("x"))
        torch.manual_seed(0)
        m = pkg.module.VGGExtractor(CIN * FQ).to(dev)
        g = torch.Generator().manual_seed(1)
        feat = torch.randn(B, T, CIN * FQ, generator=g).to(dev)
        flen = torch.full((B,), T, device=dev)
        dout = torch.randn(B, T // 4, m.out_dim, generator=g).to(dev)
        # parity of both paths against float64 (the library sequence on a float64 copy of the module)
        m64 = copy.deepcopy(m).double()
        out64 = library_forward(m64, feat.double(), flen)
        out64.backward(dout.double())
        g64 = {k: p.grad for k, p in m64.named_parameters()}
        entry = {"B": B, "T": T, "C_in": CIN, "F": FQ, "gflop_per_step": flops(B, T, FQ, CIN) / 1e9, "parity": {}}
        for path in ("gpu", "library"):
            res, grads = parity(path, m, feat, flen, dout, out64.detach())
            res["grad_max_abs_err_over_max_abs"] = max(
                float((grads[k] - g64[k]).abs().max() / g64[k].abs().max()) for k in grads)
            entry["parity"][path] = res
        del m64, out64, g64
        for path in ("gpu", "library"):                                  # warm-up of every shape and algorithm
            time_path(path, m, feat, flen, dout, 1)
        times = {"gpu": [], "library": []}
        for _ in range(args.reps):
            for path in ("gpu", "library"):
                times[path].append(time_path(path, m, feat, flen, dout, args.iters))
        for path, ts in times.items():
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            entry[path] = {"ms_median": med, "ms_min": ts[0], "ms_max": ts[-1],
                           "tflops": flops(B, T, FQ, CIN) / (med * 1e-3) / 1e12}
        entry["speedup"] = entry["library"]["ms_median"] / entry["gpu"]["ms_median"]
        # per-kernel split of the GPU path (events per C-ABI call, one separate step)
        pkg.lib.TIMER.reset()
        pkg.lib.TIMER.enabled = True
        step("gpu", m, feat, flen, dout)
        torch.cuda.synchronize()
        pkg.lib.TIMER.enabled = False
        entry["gpu_kernels_ms"] = {k: round(v["ms"], 3) for k, v in sorted(pkg.lib.TIMER.summary().items())}
        result["shapes"].append(entry)
        print(json.dumps(entry), flush=True)
        del m, feat, dout
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
