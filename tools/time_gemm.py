"""ms and TFLOP/s of the own wgmma GEMMs at the calls one cfg-B train step makes per BiLSTM layer and direction
(input projection, input gradient and the transposed weight copy it needs, dW_ih, shifted dW_hh), with the share of
the fp32-class ceiling, for both paths: 3xTF32 runs three TF32 passes, so its ceiling is a third of the data-sheet dense
TF32 rate (495 / 3 = 165 TFLOP/s on an H100 SXM at 700 W); f16x3 runs three fp16 products, a third of the data-sheet
dense fp16 rate (989 / 3 = 330 TFLOP/s), and its operand preparation passes (f16_split, and f16_split_dg: one pass
over dG of both directions; memory-bound) are timed as calls of their own.  The step runs these contractions on f16x3;
the 3xTF32 rows (through ops.gemm_tn / gemm_nn / gemm_nt) are a comparison of the two kernels at the same shapes, not calls the step makes.  Prints the card name and
power limit of the run.  QUICK=1 times layer 3 only."""
import importlib, os, subprocess, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("end-to-end-asr-pytorch_b200")
ops = pkg.ops
dev = "cuda"
CEILING = 495.0 / 3        # TFLOP/s: H100 SXM data-sheet dense TF32 / 3 passes (a data-sheet figure, not measured)
CEILING_F16 = 989.0 / 3    # TFLOP/s: H100 SXM data-sheet dense fp16 / 3 products (a data-sheet figure, not measured)
H, B = 512, 64             # cfg B: hidden size per direction, utterances per step
LAYERS = [(76672, 120), (76672, 1024), (38336, 2048), (19136, 2048)]      # (B*T rows, input width) per layer


def timeit(fn, reps=10):
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


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                    str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
print("card: %s (name, power limit)" % (q or torch.cuda.get_device_name()))
print("%-34s %6s %5s %5s %8s %8s %7s" % ("call", "M", "N", "K", "ms", "TFLOP/s", "ceiling"))
layers = LAYERS[3:] if os.environ.get("QUICK") else LAYERS
step_ms = step_tf = f16_ms = f16_prep_ms = 0.0
for li, (rows, I) in ((i, l) for i, l in enumerate(LAYERS) if l in layers):
    T = rows // B
    x = torch.randn(rows, I, device=dev)
    w = torch.randn(4 * H, I, device=dev) * 0.05
    g = torch.randn(rows, 4 * H, device=dev)
    h = torch.randn(B, T, 2 * H, device=dev)
    wlo = ops.tf32_residual(w)
    wt = w.t().contiguous()
    wtlo = ops.tf32_residual(wt)
    calls = [("L%d input projection tn (pre-split W)" % li, rows, 4 * H, I,
              lambda: ops.gemm_tn(x, w, w_lo=wlo))]
    if li > 0:                                   # the encoder input needs no gradient
        calls += [("L%d W^T copy + its residual" % li, 0, 0, 0, lambda: ops.tf32_residual(w.t().contiguous())),
                  ("L%d dX tn on W^T (pre-split)" % li, rows, I, 4 * H, lambda: ops.gemm_tn(g, wt, w_lo=wtlo)),
                  ("L%d dX nn (W in place)" % li, rows, I, 4 * H, lambda: ops.gemm_nn(g, w))]
    calls += [("L%d dW_ih nt" % li, 4 * H, I, rows, lambda: ops.gemm_nt(g, x, 4 * H, I, rows, permute_rows=True)),
              ("L%d dW_hh nt (h_prev shifted)" % li, 4 * H, H, rows,
               lambda: ops.gemm_nt(g, h, 4 * H, H, T, batches=B, a_bstride=T * 4 * H, ldb=2 * H, b_bstride=T * 2 * H,
                                   b_shift=-1, permute_rows=True))]
    for name, M, N, K, fn in calls:
        ms = timeit(fn)
        tf = 2.0 * M * N * K / ms / 1e9
        if M == 0:                               # the input gradient's weight preparation (memory-bound, no FLOPs)
            print("%-34s %26.3f" % (name, ms), flush=True)
        else:
            print("%-34s %6d %5d %5d %8.3f %8.1f %6.1f%%" % (name, M, N, K, ms, tf, 100 * tf / CEILING), flush=True)
        if "nn" not in name:                     # the step runs the tn form of dX; nn is listed for comparison
            step_ms += 2 * ms
            step_tf += 2 * 2.0 * M * N * K / 1e12
    # f16x3 as the step runs it: weight 1 = once per direction, 0.5 = once per layer (x's and X^T's images, the one
    # pass over dG of both directions, the dX contraction over both directions)
    g2 = torch.stack([g, g])
    xi, wi = ops.f16_split(x, rows, I), ops.f16_split(w, 4 * H, I)
    gts, grow, _ = ops.f16_split_dg(g2, row_images=li > 0)
    gt, wti = gts[0], None
    xt = ops.f16_split_t(x, I, rows)
    ht = ops.f16_split_t(h, H, T, batches=B, ld=2 * H, bstride=T * 2 * H, shift=-1)
    fcalls = [("L%d f16 split x (per layer)" % li, 0, 0, 0, 0.5, lambda: ops.f16_split(x, rows, I)),
              ("L%d f16 split W" % li, 0, 0, 0, 1, lambda: ops.f16_split(w, 4 * H, I)),
              ("L%d f16 input projection" % li, rows, 4 * H, I, 1, lambda: ops.gemm_f16x3(xi, wi)),
              ("L%d f16 dG prep (per layer)" % li, 0, 0, 0, 0.5, lambda: ops.f16_split_dg(g2, row_images=li > 0))]
    if li > 0:
        wti = ops.f16_split_cat_t([w, w], grow[0].shape[2] // 2)
        fcalls += [("L%d f16 split [W^T|W^T] (per layer)" % li, 0, 0, 0, 0.5,
                    lambda: ops.f16_split_cat_t([w, w], grow[0].shape[2] // 2)),
                   ("L%d f16 dX (per layer)" % li, rows, I, 8 * H, 0.5, lambda: ops.gemm_f16x3(grow, wti))]
    fcalls += [("L%d f16 split X^T (per layer)" % li, 0, 0, 0, 0.5, lambda: ops.f16_split_t(x, I, rows)),
               ("L%d f16 dW_ih" % li, 4 * H, I, rows, 1, lambda: ops.gemm_f16x3(gt, xt, permute_rows=True)),
               ("L%d f16 split h_prev^T (shifted)" % li, 0, 0, 0, 1,
                lambda: ops.f16_split_t(h, H, T, batches=B, ld=2 * H, bstride=T * 2 * H, shift=-1)),
               ("L%d f16 dW_hh" % li, 4 * H, H, rows, 1, lambda: ops.gemm_f16x3(gt, ht, permute_rows=True))]
    for name, M, N, K, wgt, fn in fcalls:
        ms = timeit(fn)
        if M == 0:
            print("%-34s %26.3f" % (name, ms), flush=True)
            f16_prep_ms += 2 * wgt * ms
        else:
            tf = 2.0 * M * N * K / ms / 1e9
            print("%-34s %6d %5d %5d %8.3f %8.1f %6.1f%%" % (name, M, N, K, ms, tf, 100 * tf / CEILING_F16), flush=True)
            f16_ms += 2 * wgt * ms
    del x, w, g, g2, h, wlo, wt, wtlo, xi, wi, wti, gts, grow, gt, xt, ht
print("sum over both directions: %.1f ms for %.2f TFLOP = %.1f TFLOP/s (%.1f%% of the %.0f TFLOP/s ceiling)"
      % (step_ms, step_tf, step_tf / step_ms * 1e3, 100 * step_tf / step_ms * 1e3 / CEILING, CEILING))
print("f16x3, both directions: GEMMs %.1f ms = %.1f TFLOP/s (%.1f%% of the %.0f TFLOP/s ceiling), preparation passes "
      "%.1f ms, together %.1f ms" % (f16_ms, step_tf / f16_ms * 1e3, 100 * step_tf / f16_ms * 1e3 / CEILING_F16,
                                      CEILING_F16, f16_prep_ms, f16_ms + f16_prep_ms))
