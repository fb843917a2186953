"""The GRU encoder layer on the persistent recurrence kernels (ops.BiGRUFn) against the library nn.GRU (cuDNN, TF32
off), on one H100, in one process:

  1. one bidirectional layer, forward + backward, at the cfg-B encoder shapes (B 64, H 512): layer 0 (T 1198, I 120)
     and the two upper layers (T 599 / 299, I 2048).  Repetitions of the two arms are interleaved; ms median and range,
     the kernel split of our layer (recurrence vs layer GEMMs) and the largest output / dx difference between the arms.
  2. a whole cfg-B train step with `encoder.module: GRU` through TrainStep with CUDA-graph replay, our layers against
     the same model with its GRU layers on nn.GRU (graph replay too where cuDNN's RNN can be captured, else eager,
     which is stated).
The card's name and power limit are read in the same run.  env: REPS (5), ITERS (3), STEPS (10), PARTS (layer,step).
"""
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")
L = pkg.lib
REPS = int(os.environ.get("REPS", 5))
ITERS = int(os.environ.get("ITERS", 3))
STEPS = int(os.environ.get("STEPS", 10))
PARTS = os.environ.get("PARTS", "layer,step").split(",")
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
assert torch.cuda.is_available(), "time_gru.py measures on the GPU"
DEV = torch.device("cuda")


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # noqa: BLE001 - reported, not hidden
        pl = "unknown (%s)" % e
    return {"card": torch.cuda.get_device_name(0), "power_limit": pl}


def summary(ts):
    return {"median_ms": round(statistics.median(ts), 3), "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3),
            "n": len(ts)}


def timed(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def layer_part():
    out = []
    for B, T, I, H in ((64, 1198, 120, 512), (64, 599, 2048, 512), (64, 299, 2048, 512)):
        torch.manual_seed(0)
        layer = pkg.module.RNNLayer(I, "GRU", H, True, 0, False, 1, "drop", False).to(DEV)
        x = torch.randn(B, T, I, device=DEV, requires_grad=True)
        gy = torch.randn(B, T, 2 * H, device=DEV)
        lens = torch.full((B,), T)

        def own():
            x.grad = None
            y, _ = layer(x, lens)
            y.backward(gy)
            return y

        def lib():
            x.grad = None
            y, _ = layer.layer(x)
            y.backward(gy)
            return y

        arms = {"own": own, "nn.GRU": lib}
        res = {}
        for name, fn in arms.items():                      # warm-up, outputs for the comparison
            for _ in range(2):
                y = fn()
            torch.cuda.synchronize()
            res[name] = (y.detach().clone(), x.grad.detach().clone())
        ts = {name: [] for name in arms}
        for _ in range(REPS):
            for name, fn in arms.items():
                ts[name].append(timed(fn, ITERS))
        L.TIMER.enabled = True
        L.TIMER.reset()
        own()
        torch.cuda.synchronize()
        L.TIMER.enabled = False
        split = {k: round(v["ms"], 3) for k, v in sorted(L.TIMER.summary().items())}
        rec = sum(v for k, v in split.items() if k.startswith("bigru"))
        gemm = sum(v for k, v in split.items() if k.startswith(("gemm", "f16_split", "split_tf32")))
        r = {"shape": "B %d T %d I %d -> H %d, bidirectional, forward + backward" % (B, T, I, H),
             "own": summary(ts["own"]), "nn.GRU (cuDNN, TF32 off)": summary(ts["nn.GRU"]),
             "own_kernel_ms": split, "own_recurrence_ms": round(rec, 3), "own_layer_gemm_ms": round(gemm, 3),
             # the layer GEMMs run on 4H packed rows of which H are zero in each weight: a quarter of their time
             "zero_slot_share_ms": round(gemm / 4, 3),
             "max_abs_dy": float((res["own"][0] - res["nn.GRU"][0]).abs().max()),
             "max_abs_y": float(res["nn.GRU"][0].abs().max()),
             "max_abs_ddx": float((res["own"][1] - res["nn.GRU"][1]).abs().max()),
             "max_abs_dx": float(res["nn.GRU"][1].abs().max())}
        print(json.dumps(r), flush=True)
        out.append(r)
        del layer, x, gy
        torch.cuda.empty_cache()
    return out


def step_part():
    cfg = pkg.synthetic.load_config("cfgB")
    cfg["model"]["encoder"] = dict(cfg["model"]["encoder"], module="GRU")
    vocab = cfg["data"]["corpus"]["vocab_size"]
    B = cfg["data"]["corpus"]["batch_size"]
    waves, lens, txt = pkg.synthetic.make_batch(vocab, B, 192000, seed=1000)
    wave, lens, txt = waves.to(DEV), lens.to(DEV), txt.to(DEV)
    supported = pkg.ops.rnn_layer_supported
    arms, graphed = {}, {}
    for name, own in (("own", True), ("nn.GRU", False)):
        pkg.ops.rnn_layer_supported = supported if own else (lambda *a: False)
        step = pkg.TrainStep(cfg, vocab, device=DEV, seed=0)
        ok = step.capture(wave, lens, txt, warmup=3)
        graphed[name] = bool(ok) or ("eager: %s" % step.graph_error)
        if not ok:
            for _ in range(3):
                step(wave, lens, txt)
        arms[name] = (step, own)
    pkg.ops.rnn_layer_supported = supported
    ts = {name: [] for name in arms}
    for _ in range(REPS):
        for name, (step, own) in arms.items():
            pkg.ops.rnn_layer_supported = supported if own else (lambda *a: False)
            ts[name].append(timed(lambda: step(wave, lens, txt), STEPS))
    pkg.ops.rnn_layer_supported = supported
    r = {"workload": "cfgB (B %d, 192000 samples) with encoder.module GRU, whole train step" % B,
         "own": summary(ts["own"]), "nn.GRU (cuDNN, TF32 off)": summary(ts["nn.GRU"]), "graph_replay": graphed}
    print(json.dumps(r), flush=True)
    return r


def main():
    res = {"device": card(), "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    print(json.dumps(res["device"]), flush=True)
    if "layer" in PARTS:
        res["layer"] = layer_part()
    if "step" in PARTS:
        res["step"] = step_part()
    res["device_after"] = card()
    out = os.environ.get("OUT")
    if out:
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
