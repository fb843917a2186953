"""ms / effective TFLOP/s of the own wgmma 3xTF32 GEMM forms (tn, nn, nt) at the cfg-B layer shapes, next to the cuBLAS
3xTF32 composition (3 library GEMMs + split passes) and a single cuBLAS TF32 GEMM (not fp32-class; speed reference)."""
import importlib, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")
ops = pkg.ops
dev = "cuda"


def timeit(fn, reps=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def lib3(a, b_t):
    return ops.mm3(ops.Split(a), ops.Split(b_t))


def tf32(a, b):
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        return a @ b
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False


shapes = [(76672, 2048, 120), (38336, 2048, 2048), (19168, 2048, 2048), (9584, 2048, 2048)]
if os.environ.get("QUICK"):
    shapes = shapes[1:2]
for M, N, K in shapes:
    x = torch.randn(M, K, device=dev)
    w = torch.randn(N, K, device=dev) * 0.05
    dy = torch.randn(M, N, device=dev)
    fl = 2.0 * M * N * K / 1e9
    t = timeit(lambda: ops.gemm_tn(x, w))
    wlo = ops.tf32_residual(w)
    tp = timeit(lambda: ops.gemm_tn(x, w, w_lo=wlo))
    print("tn  pre-split W                              own %7.3f ms (%6.1f TF)" % (tp, fl / tp), flush=True)
    xlo = ops.tf32_residual(x)
    tp = timeit(lambda: ops.gemm_tn(x, w, w_lo=wlo, a_lo=xlo))
    print("tn  both operands pre-split                  own %7.3f ms (%6.1f TF)" % (tp, fl / tp), flush=True)
    tp = timeit(lambda: ops.tf32_residual(dy))
    print("    residual pass over dy [%d x %d]          %7.3f ms" % (M, N, tp), flush=True)
    del xlo
    t2 = timeit(lambda: lib3(x, w.t()))
    t3 = timeit(lambda: tf32(x, w.t()))
    print("tn  y=x.W^T   M=%6d N=%5d K=%5d  own %7.3f ms (%6.1f TF)  cublas3x %7.3f ms  cublas-tf32x1 %7.3f ms" % (M, N, K, t, fl / t, t2, t3), flush=True)
    t = timeit(lambda: ops.gemm_nn(dy, w))
    t2 = timeit(lambda: lib3(dy, w))
    print("nn  dx=dy.W   M=%6d N=%5d K=%5d  own %7.3f ms (%6.1f TF)  cublas3x %7.3f ms" % (M, K, N, t, fl / t, t2), flush=True)
    t = timeit(lambda: ops.gemm_nt(dy, x, N, K, M))
    t2 = timeit(lambda: lib3(dy.t(), x))
    print("nt  dW=dy^T.x M=%6d N=%5d K=%5d  own %7.3f ms (%6.1f TF)  cublas3x %7.3f ms" % (N, K, M, t, fl / t, t2), flush=True)
