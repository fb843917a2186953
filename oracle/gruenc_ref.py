"""CPU ORACLE (test infrastructure, NOT a product path) for the GRU encoder layer (encoder.module: GRU): a float64
restatement of the persistent (Bi)GRU recurrence at the C ABI of b200asr_bigru_fwd / _bwd, in the layout of
oracle/lstm_ref.recurrence.  The cell is oracle/gru_ref.gru_cell's (ATen's GRUCell expression order) on the packed
4-slot gate layout of ops.pack_decoder_weights("GRU").
"""
import torch


def recurrence(pre, whh, dout=None, dtype=torch.float64):
    """The GRU recurrence in `dtype` on the CPU: (out, hstate, gates, dG); dG is None without `dout`.
    pre [ndir, B, T, H, 4] = the packed input projection (gi_r + b_hr, gi_z + b_hz, gi_n, b_hn) per unit, whh [ndir, 4H,
    H] packed [W_hr; W_hz; 0; W_hn] (gate-major rows), dout [B, T, ndir*H]; direction 1 runs in reverse time, zero
    initial state.  gates = (r, z, n, gh_n), hstate [ndir, B, T, H] = h after every step, dG = d(sum(out * dout)) /
    d(pre) in pre's layout."""
    ndir, B, T, H, _ = pre.shape
    p = pre.detach().to("cpu", dtype).clone().requires_grad_(dout is not None)
    w = whh.detach().to("cpu", dtype)
    outs, gts = [], []
    for d in range(ndir):
        frames = p[d].unbind(1)
        h = torch.zeros(B, H, dtype=dtype)
        o_t, g_t = [None] * T, [None] * T
        for step in range(T):
            t = step if d == 0 else T - 1 - step
            a = frames[t] + (h @ w[d].t()).view(B, 4, H).transpose(1, 2)
            r, z = torch.sigmoid(a[..., 0]), torch.sigmoid(a[..., 1])
            n = torch.tanh(a[..., 2] + r * a[..., 3])
            h = (h - n) * z + n
            o_t[t], g_t[t] = h, torch.stack([r, z, n, a[..., 3]], -1)
        outs.append(torch.stack(o_t, 1))
        gts.append(torch.stack(g_t, 1))
    out = torch.cat(outs, -1)
    dG = None
    if dout is not None:
        (out * dout.detach().to("cpu", dtype)).sum().backward()
        dG = p.grad.detach()
    return out.detach(), torch.stack(outs).detach(), torch.stack(gts).detach(), dG
